"""Completing tokens without a GPU: the brute-force model against the oracle (a completing id is one whose append makes a
Standard overlapping match end at the new last token), the image interpreter of acb_completions_write's bytes against
the model, the token format's inverse through the builder, the C ABI's argument checks and exports, and the Python
argument errors that need no device."""
import ctypes as C

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import MatchKind, TokenAhoCorasick, _capi
from oracle import Oracle

from .completions_model import (ALPHA, LIMIT, ComplImage, build_automaton, encode, image_bytes, model_completing,
                                random_patterns)


def _histories(rng, pats, alphabet, n):
    """Random histories, half of them ending in some pattern's p[:-1] (so that it completes), some empty."""
    out = [[]]
    for i in range(n):
        h = [int(x) for x in rng.choice(alphabet, int(rng.integers(0, 12)))]
        if i % 2 and pats:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        out.append(h)
    return out


def _subsets(rng, n_pats):
    return [None, set(), {p for p in range(n_pats) if rng.random() < 0.3}, {p for p in range(n_pats) if rng.random() < 0.8}]


# ---- the model against the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_model_equals_oracle(seed):
    rng = np.random.default_rng(seed)
    alphabet = np.array(ALPHA if seed % 2 else [3, 4, 5])
    pats = random_patterns(rng, int(rng.integers(1, 10)), 4, alphabet)
    hists = _histories(rng, pats, alphabet, 10)
    for S in _subsets(rng, len(pats)):
        admitted = [p for i, p in enumerate(pats) if S is None or i in S]
        orc = Oracle([encode(p) for p in admitted], "Standard") if admitted else None
        for h in hists:
            want = model_completing(pats, h, S)
            if orc is None:
                assert want == []
                continue
            extra = [int(x) for x in rng.choice(alphabet, 4)] + [int(ALPHA[-1]), 0]
            for t in sorted(set(want) | set(extra)):
                ends = {e for _, _, e in orc.find(encode(h + [t]), overlapping=True)}
                assert (t in want) == (3 * (len(h) + 1) in ends), (h, t, S)


def test_model_ignores_history_beyond_k_minus_one():
    pats = [[1, 2, 3], [9]]
    assert model_completing(pats, [7, 7, 7, 1, 2]) == [3, 9]
    assert model_completing(pats, [1, 2, 7]) == [9]
    assert model_completing(pats, [2]) == [9]
    assert model_completing([], [1, 2]) == []


# ---- the image interpreter against the model -------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_image_interpreter_equals_model(seed):
    rng = np.random.default_rng(100 + seed)
    alphabet = np.array(ALPHA if seed % 2 else [3, 4, 5, 6])
    pats = random_patterns(rng, int(rng.integers(1, 30)), 1 + seed % 5, alphabet)
    img = ComplImage(image_bytes(pats))
    img.check_structure(pats)
    hists = _histories(rng, pats, alphabet, 20)
    hists.append([-1, LIMIT, 1 << 40] + (pats[0][:-1] if pats else []))   # ids no pattern token equals
    hists.append(pats[0][:-1] + [-5])
    for S in _subsets(rng, len(pats)):
        for h in hists:
            want = model_completing(pats, h, S)
            assert img.completing(h, S) == want, (h, S)
            got = img.emitted(h, S)
            assert sorted(got) == want and len(set(got)) == len(got), (h, S)


def test_image_of_no_patterns_and_one_token_patterns():
    img = ComplImage(image_bytes([]))
    img.check_structure([])
    assert (img.n_nodes, img.n_entries, img.depth, img.max_last) == (1, 0, 0, 0)
    assert img.completing([1, 2, 3]) == []
    pats = [[7], [3], [7], [5]]
    img = ComplImage(image_bytes(pats))
    img.check_structure(pats)
    assert (img.n_nodes, img.depth, img.max_last) == (1, 0, 7)
    assert img.node_entries(0) == [(3, 1), (5, 3), (7, 0), (7, 2)]
    assert img.completing([]) == [3, 5, 7] and img.emitted([9, 9]) == [3, 5, 7]
    assert img.emitted([], {2, 3}) == [5, 7] and img.completing([], set()) == []


def test_image_root_with_many_children_and_a_long_pattern():
    rng = np.random.default_rng(7)
    pats = [[int(a), int(b)] for a, b in zip(rng.permutation(40000), rng.integers(0, 50, 40000))]
    long_pat = [int(x) for x in rng.choice(ALPHA, 210)]
    pats.append(long_pat)
    img = ComplImage(image_bytes(pats))
    assert int(img.nodes[0, 1]) > 32768 and img.depth == 209
    for h in ([0], [39999], [12345, 3], long_pat[:-1], [5] + long_pat[:-1], long_pat[:-2]):
        assert img.completing(h) == model_completing(pats, h)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_image_does_not_depend_on_the_match_kind(kind):
    pats = [[1, 2], [2], [1, 2, 3], [1, 2]]
    assert image_bytes(pats, kind) == image_bytes(pats, 0)


# ---- the token format's inverse --------------------------------------------------------------------------------------
def test_token_decode_inverts_token_code_at_the_edge_ids():
    """Every edge id encoded by acb_tokens_encode_host (token_code) comes back out of the builder (token_decode): as a
    child token (a non-last position) and as an entry token (a last one)."""
    pats = [[a, b] for a in ALPHA for b in ALPHA]
    enc = []
    for p in pats:
        ids = np.asarray(p, dtype=np.int64)
        out = np.empty(6, dtype=np.uint8)
        bad = np.full(1, (1 << 64) - 1, dtype=np.uint64)
        assert _capi.lib().acb_tokens_encode_host(ids.ctypes.data, 8, 2, out.ctypes.data, bad.ctypes.data) == _capi.ACB_OK
        assert out.tobytes() == encode(p)
        enc.append(out.tobytes())
    L, h = build_automaton(enc)
    try:
        n = C.c_uint64(0)
        assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_OK
        buf = np.zeros(n.value, dtype=np.uint8)
        assert L.acb_completions_write(h, buf.ctypes.data, n.value) == _capi.ACB_OK
    finally:
        L.acb_free(h)
    img = ComplImage(buf.tobytes())
    img.check_structure(pats)
    assert sorted(int(t) for t in img.kid_tok[1:]) == sorted(set(ALPHA))
    assert sorted({int(t) for t, _ in img.entries}) == sorted(set(ALPHA)) and img.max_last == LIMIT - 1


@pytest.mark.parametrize("bad", [b"ab", b"\x80\x00\x00\x80", bytes([0x00, 0x00, 0x00]), bytes([0x80, 0x80, 0x00]),
                                 bytes([0x80, 0x00, 0x80]), bytes([0x81, 0x00, 0x00, 0x05, 0x00, 0x00])])
def test_build_refuses_patterns_not_in_the_token_format(bad):
    L, h = build_automaton([encode([1, 2]), bad])
    try:
        n = C.c_uint64(0)
        assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_EINVAL
        assert "token format" in _capi.last_error()
        buf = np.zeros(64, dtype=np.uint8)
        assert L.acb_completions_write(h, buf.ctypes.data, 64) == _capi.ACB_EINVAL   # nothing was built
    finally:
        L.acb_free(h)


# ---- the C ABI -------------------------------------------------------------------------------------------------------
CALLS = ["acb_completions_build", "acb_completions_write", "acb_completions_describe", "acb_completions_count",
         "acb_completions_emit", "acb_completions_mask"]


def test_exports():
    L = _capi.lib()
    for name in CALLS:
        assert name in _capi.EXPORTS
        assert hasattr(L, name)


def test_build_write_describe_errors():
    L = _capi.lib()
    n = C.c_uint64(0)
    assert L.acb_completions_build(None, C.byref(n)) == _capi.ACB_EINVAL
    Lb, h = build_automaton([encode([1, 2, 3]), encode([4])])
    try:
        assert L.acb_completions_build(h, None) == _capi.ACB_EINVAL
        buf = np.zeros(1024, dtype=np.uint8)
        assert L.acb_completions_write(h, buf.ctypes.data, 1024) == _capi.ACB_EINVAL   # not built yet
        assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_OK and 0 < n.value <= 1024
        assert L.acb_completions_write(h, None, 1024) == _capi.ACB_EINVAL
        assert L.acb_completions_write(h, buf.ctypes.data, n.value - 1) == _capi.ACB_ECAPACITY
        assert L.acb_completions_write(h, buf.ctypes.data, n.value) == _capi.ACB_OK
        d = _capi.CompletionsDesc()
        assert L.acb_completions_describe(buf.ctypes.data, C.byref(d)) == _capi.ACB_OK
        assert (d.nodes, d.entries, d.depth, d.max_last) == (3, 2, 2, 4)
        assert L.acb_completions_describe(buf.ctypes.data, None) == _capi.ACB_EINVAL
        assert L.acb_completions_describe(None, C.byref(d)) == _capi.ACB_EINVAL
        junk = np.zeros(64, dtype=np.uint8)
        assert L.acb_completions_describe(junk.ctypes.data, C.byref(d)) == _capi.ACB_EINVAL
    finally:
        Lb.acb_free(h)


P = 0x3000   # never dereferenced: every refusal below happens before any device work


def _filter(**kw):
    f = _capi.PatternFilter()
    f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = P, 1, P, 4
    for k, v in kw.items():
        setattr(f, k, v)
    return C.byref(f)


COMMON_BAD = {
    "a": dict(a=None), "image": dict(image=None), "tokens": dict(tokens=None), "offsets": dict(offsets=None),
    "width3": dict(width=3), "width0": dict(width=0), "n_tokens": dict(n_tokens=1 << 60), "rows_neg": dict(rows=-1),
    "rows_high": dict(rows=1 << 32), "filter_sets": dict(filter=_filter(n_sets=0)), "filter_bits": dict(filter=_filter(dev_set_bits=None)),
    "filter_width": dict(filter=_filter(index_bytes=2)), "filter_index": dict(filter=_filter(dev_set_index=None)),
}


def _call(L, mode, h, **over):
    a = dict(a=h, image=P, tokens=P, width=8, n_tokens=10, offsets=P, rows=2, filter=None, out=P, row_offsets=P,
             logits=P, dtype=_capi.ACB_LOGITS_BF16, stride=200, vocab=100, value=float("-inf"))
    a.update(over)
    head = (a["a"], a["image"], a["tokens"], a["width"], a["n_tokens"], a["offsets"], a["rows"])
    if mode == "count":
        return L.acb_completions_count(*head, a["out"], a["filter"], None)
    if mode == "emit":
        return L.acb_completions_emit(*head, a["row_offsets"], a["out"], a["filter"], None)
    return L.acb_completions_mask(*head, a["logits"], a["dtype"], a["stride"], a["vocab"], a["value"], a["filter"], None)


@pytest.fixture
def built():
    L, h = build_automaton([encode([1, 2, 3]), encode([40, 50]), encode([7])])
    n = C.c_uint64(0)
    assert L.acb_completions_build(h, C.byref(n)) == _capi.ACB_OK
    yield L, h
    L.acb_free(h)


@pytest.mark.parametrize("mode", ["count", "emit", "mask"])
@pytest.mark.parametrize("bad", sorted(COMMON_BAD))
def test_einval_common(built, mode, bad):
    L, h = built
    assert _call(L, mode, h, **COMMON_BAD[bad]) == _capi.ACB_EINVAL, _capi.last_error()


@pytest.mark.parametrize("mode,bad", [("count", dict(out=None)), ("emit", dict(out=None)), ("emit", dict(row_offsets=None)),
                                      ("mask", dict(logits=None)), ("mask", dict(dtype=3)), ("mask", dict(dtype=-1)),
                                      ("mask", dict(vocab=0)), ("mask", dict(vocab=-5)), ("mask", dict(vocab=1 << 62)),
                                      ("mask", dict(stride=-1)), ("mask", dict(stride=1 << 62)), ("mask", dict(vocab=50)),
                                      ("mask", dict(vocab=40))])
def test_einval_per_mode(built, mode, bad):
    L, h = built
    assert _call(L, mode, h, **bad) == _capi.ACB_EINVAL, _capi.last_error()


@pytest.mark.parametrize("mode", ["count", "emit", "mask"])
def test_einval_before_build(mode):
    L, h = build_automaton([encode([1, 2])])
    try:
        assert _call(L, mode, h) == _capi.ACB_EINVAL
        assert "acb_completions_build" in _capi.last_error()
    finally:
        L.acb_free(h)


def test_vocab_refusal_names_the_largest_last_id(built):
    L, h = built
    assert _call(L, "mask", h, vocab=50) == _capi.ACB_EINVAL
    assert "50" in _capi.last_error()


# ---- Python argument errors that need no device ----------------------------------------------------------------------
def test_host_forms_check_ids_first():
    tac = TokenAhoCorasick([[1, 2], [3]])
    with pytest.raises(ValueError, match=r"history 0: token 1 = -1 is outside \[0, 2097152\)"):
        tac.completing_tokens([5, -1, 2])
    with pytest.raises(ValueError, match=r"history 1: token 0 = 2097152"):
        tac.completing_tokens_batch([[1], [1 << 21]])
    with pytest.raises(TypeError):
        tac.completing_tokens([1.5, 2.0])
    with pytest.raises(TypeError):
        tac.completing_tokens([[1, 2], [3, 4]])
    with pytest.raises(ValueError, match="one set of pattern ids per haystack"):
        tac.completing_tokens_batch([[1], [2]], patterns=[[0]])
    assert tac.completing_tokens_batch([]) == []


def test_device_forms_refuse_host_tensors():
    tac = TokenAhoCorasick([[1, 2], [3]])
    offs = torch.tensor([0, 2], dtype=torch.int64)
    for bad in (torch.tensor([1, 2], dtype=torch.int64), [1, 2], torch.tensor([1.0, 2.0])):
        with pytest.raises(TypeError, match="tokens must be a 1-D CUDA tensor"):
            tac.completing_tokens_device(bad, offs)
        with pytest.raises(TypeError, match="tokens must be a 1-D CUDA tensor"):
            tac.mask_completing_tokens_(torch.zeros(1, 8), bad, offs)


def test_token_matchkinds_share_the_host_answer_model():
    """The contract does not depend on the match kind: the model has no kind, and the images are equal."""
    pats = [[1, 2], [2, 3], [1]]
    assert model_completing(pats, [1]) == [1, 2]
    for kind in MatchKind:
        assert image_bytes(pats, kind.value) == image_bytes(pats, 0)
