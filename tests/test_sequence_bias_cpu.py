"""Per-pattern biases for completing tokens without a GPU: the brute-force model of the contract's sum order, the image
interpreter that runs the bias kernel's algorithm against it bit for bit, a case where the order decides the float32
result, acb_completions_bias's argument checks and export, and the Python argument errors that need no device."""
import ctypes as C

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import TokenAhoCorasick, _capi

from .completions_model import ALPHA, LIMIT, ComplImage, build_automaton, encode, image_bytes, model_completing, random_patterns
from .sequence_bias_model import BiasModel, apply_sums, interp_bias_sums, model_bias_sums


def _histories(rng, pats, alphabet, n):
    """Random histories, half of them ending in some pattern's p[:-1], some empty, some with ids no pattern holds."""
    out = [[]]
    for i in range(n):
        h = [int(x) for x in rng.choice(alphabet, int(rng.integers(0, 12)))]
        if i % 2 and pats:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        out.append(h)
    if pats:
        out.append([-1, LIMIT, 1 << 40] + pats[0][:-1])
        out.append(pats[-1][:-1] + [-5])
    return out


def _subsets(rng, n_pats):
    return [None, set(), {p for p in range(n_pats) if rng.random() < 0.3}, {p for p in range(n_pats) if rng.random() < 0.8}]


def _bits(d):
    return {t: np.float32(s).view(np.uint32) for t, s in d.items()}


# ---- the model -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_model_keys_are_the_completing_ids(seed):
    rng = np.random.default_rng(200 + seed)
    alphabet = np.array(ALPHA if seed % 2 else [3, 4, 5])
    pats = random_patterns(rng, int(rng.integers(1, 20)), 4, alphabet)
    bias = rng.standard_normal(len(pats)).astype(np.float32)
    fast = BiasModel(pats)
    for S in _subsets(rng, len(pats)):
        for h in _histories(rng, pats, alphabet, 15):
            got = model_bias_sums(pats, h, bias, S)
            assert sorted(got) == model_completing(pats, h, S)
            assert _bits(fast(h, bias, S)) == _bits(got)


def test_model_sums_longest_first_then_by_pid():
    # id 9 is completed by [9] (pid 0), [1, 9] (pids 1 and 3) and [2, 1, 9] (pid 2): order 2, 1, 3, 0
    pats = [[9], [1, 9], [2, 1, 9], [1, 9], [4]]
    bias = np.array([1.0, 1e8, -1e8, 1.0, 0.5], dtype=np.float32)
    got = model_bias_sums(pats, [2, 1], bias)
    # -1e8 + 1e8 = 0, + 1 = 1, + 1 = 2; any order that adds a 1 next to a 1e8 loses it
    assert got == {9: np.float32(2.0), 4: np.float32(0.5)}
    assert model_bias_sums(pats, [1], bias)[9] == np.float32(1e8) + np.float32(1.0) + np.float32(1.0)
    assert model_bias_sums(pats, [7], bias) == {9: np.float32(1.0), 4: np.float32(0.5)}


def test_order_decides_the_float32_result():
    """Biases 1e8, 1, -1e8 at three depths: the contract's order (longest first) gives 1e8 - 1e8 + 1 = 1 when the
    -1e8 pattern is the longest, and 0 when the 1 comes between them."""
    pats = [[5], [3, 5], [2, 3, 5]]
    img = ComplImage(image_bytes(pats))
    for bias, want in (([1.0, 1e8, -1e8], 1.0), ([1e8, 1.0, -1e8], 0.0), ([-1e8, 1.0, 1e8], 0.0), ([1.0, -1e8, 1e8], 1.0)):
        b = np.array(bias, dtype=np.float32)
        assert model_bias_sums(pats, [2, 3], b) == {5: np.float32(want)}, bias
        assert _bits(interp_bias_sums(img, [2, 3], b)) == _bits({5: want}), bias
    # a naive sum from 0.0 in pid order would differ from the contract's in the first two cases
    assert np.float32(np.float32(np.float32(0) + np.float32(1.0)) + np.float32(1e8)) + np.float32(-1e8) == 0.0


def test_sum_starts_from_the_first_term():
    """A lone -0.0 bias stays -0.0, so a -0.0 logit stays -0.0 (0.0 + -0.0 would be +0.0)."""
    pats = [[5], [6], [6]]
    bias = np.array([-0.0, -0.0, -0.0], dtype=np.float32)
    for s in (model_bias_sums(pats, [], bias), interp_bias_sums(ComplImage(image_bytes(pats)), [], bias)):
        assert {t: np.signbit(v) for t, v in s.items()} == {5: True, 6: True}
    logits = torch.tensor([[0.0, -0.0, 0.0, 0.0, 0.0, -0.0, -0.0]], dtype=torch.float32)
    out = apply_sums(logits, [model_bias_sums(pats, [], bias)])
    assert torch.equal(out.view(torch.int32), logits.view(torch.int32))


# ---- the image interpreter against the model, bit for bit ------------------------------------------------------------
@pytest.mark.parametrize("seed", range(10))
def test_interpreter_equals_model(seed):
    rng = np.random.default_rng(300 + seed)
    alphabet = np.array(ALPHA if seed % 2 else [3, 4, 5, 6])
    pats = random_patterns(rng, int(rng.integers(1, 40)), 1 + seed % 5, alphabet)
    pats += [list(pats[0]), list(pats[-1]), [int(alphabet[0])], [int(alphabet[0])]]   # more duplicates, one-token patterns
    img = ComplImage(image_bytes(pats))
    img.check_structure(pats)
    # random, not dyadic: the sums round, so any other order would show
    bias = (rng.standard_normal(len(pats)) * 10.0 ** rng.integers(-3, 6, len(pats))).astype(np.float32)
    for S in _subsets(rng, len(pats)):
        for h in _histories(rng, pats, alphabet, 25):
            want = model_bias_sums(pats, h, bias, S)
            assert _bits(interp_bias_sums(img, h, bias, S)) == _bits(want), (h, S)


def test_interpreter_many_patterns_share_a_last_token():
    rng = np.random.default_rng(11)
    pats = [[int(x) for x in rng.choice([1, 2, 3], int(rng.integers(0, 5)))] + [7] for _ in range(200)]
    img = ComplImage(image_bytes(pats))
    bias = rng.standard_normal(len(pats)).astype(np.float32) * np.float32(1000.0)
    for h in ([], [1], [3, 2, 1], [1, 1, 1, 1], [2, 2, 3, 1, 2]):
        for S in (None, set(range(0, 200, 3))):
            want = model_bias_sums(pats, h, bias, S)
            assert set(want) <= {7}
            assert _bits(interp_bias_sums(img, h, bias, S)) == _bits(want)


def test_apply_sums_rounds_once_to_the_logits_dtype():
    # 1 + 2^-9 + 2^-9 in bf16 (8 bits of mantissa): each step alone rounds back to 1, the float32 sum rounds up
    logits = torch.ones(1, 3, dtype=torch.bfloat16)
    out = apply_sums(logits, [{1: np.float32(2.0 ** -8) + np.float32(2.0 ** -10)}])
    assert out[0, 1].item() == 1.0 + 2.0 ** -7 and out[0, 0].item() == 1.0 and out[0, 2].item() == 1.0
    half = apply_sums(torch.zeros(1, 2, dtype=torch.float16), [{0: np.float32(70000.0)}])
    assert torch.isinf(half[0, 0]) and half[0, 1].item() == 0.0


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_export():
    assert "acb_completions_bias" in _capi.EXPORTS
    assert hasattr(_capi.lib(), "acb_completions_bias")


P = 0x3000   # never dereferenced: every refusal below happens before any device work


def _filter(**kw):
    f = _capi.PatternFilter()
    f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = P, 1, P, 4
    for k, v in kw.items():
        setattr(f, k, v)
    return C.byref(f)


def _call(L, h, **over):
    a = dict(a=h, image=P, tokens=P, width=8, n_tokens=10, offsets=P, rows=2, bias=P, logits=P, dtype=_capi.ACB_LOGITS_BF16,
             stride=200, vocab=100, filter=None)
    a.update(over)
    return L.acb_completions_bias(a["a"], a["image"], a["tokens"], a["width"], a["n_tokens"], a["offsets"], a["rows"], a["bias"],
                                  a["logits"], a["dtype"], a["stride"], a["vocab"], a["filter"], None)


BAD = {
    "a": dict(a=None), "image": dict(image=None), "tokens": dict(tokens=None), "offsets": dict(offsets=None),
    "width3": dict(width=3), "width0": dict(width=0), "n_tokens": dict(n_tokens=1 << 60), "rows_neg": dict(rows=-1),
    "rows_high": dict(rows=1 << 32), "filter_sets": dict(filter=_filter(n_sets=0)), "filter_bits": dict(filter=_filter(dev_set_bits=None)),
    "filter_width": dict(filter=_filter(index_bytes=2)), "filter_index": dict(filter=_filter(dev_set_index=None)),
    "logits": dict(logits=None), "dtype3": dict(dtype=3), "dtype_neg": dict(dtype=-1), "vocab0": dict(vocab=0),
    "vocab_neg": dict(vocab=-5), "vocab_high": dict(vocab=1 << 62), "stride_neg": dict(stride=-1), "stride_high": dict(stride=1 << 62),
    "vocab_max_last": dict(vocab=50), "vocab_below": dict(vocab=40), "bias": dict(bias=None),
}


@pytest.fixture
def built():
    L, h = build_automaton([encode([1, 2, 3]), encode([40, 50]), encode([7])])
    n = C.c_uint64(0)
    assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_OK
    yield L, h
    L.acb_free(h)


@pytest.mark.parametrize("bad", sorted(BAD))
def test_einval(built, bad):
    L, h = built
    assert _call(L, h, **BAD[bad]) == _capi.ACB_EINVAL, _capi.last_error()


def test_einval_before_build():
    L, h = build_automaton([encode([1, 2])])
    try:
        assert _call(L, h) == _capi.ACB_EINVAL
        assert "acb_completions_build" in _capi.last_error()
    finally:
        L.acb_free(h)


def test_null_pointers_allowed_without_rows(built):
    """n_rows == 0 needs no per-row pointer; the refusals above all come before the device is touched, so this is
    the only call here that may reach the device query (and on a machine without one it fails there, not earlier)."""
    L, h = built
    rc = _call(L, h, rows=0, offsets=None, bias=None, logits=None)
    assert rc in (_capi.ACB_OK, _capi.ACB_ECUDA), _capi.last_error()


def test_vocab_refusal_names_the_largest_last_id(built):
    L, h = built
    assert _call(L, h, vocab=50) == _capi.ACB_EINVAL
    assert "50" in _capi.last_error()


# ---- Python argument errors that need no device ----------------------------------------------------------------------
def test_refuses_host_tensors():
    tac = TokenAhoCorasick([[1, 2], [3]])
    offs = torch.tensor([0, 2], dtype=torch.int64)
    for bad in (torch.tensor([1, 2], dtype=torch.int64), [1, 2], torch.tensor([1.0, 2.0])):
        with pytest.raises(TypeError, match="tokens must be a 1-D CUDA tensor"):
            tac.bias_completing_tokens_(torch.zeros(1, 8), bad, offs, torch.zeros(2))
