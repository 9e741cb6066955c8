"""Vocabulary stop strings without a GPU: the image interpreter (what vocab_stop_kernel does) against the brute force
over the oracle on the seeded vocabulary families, the new = 1 identity with the completing-token brute force, the C
ABI's argument checks and export, and the Python argument errors that need no device."""
import ctypes as C

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import BytesAhoCorasick, _capi

from . import vocab_families as vf
from .test_vocab_cpu import CASES, _case
from .vocab_model import BruteModel, build_automaton, image_bytes
from .vocab_stop_model import BruteStop, StopImage


def _news(h):
    return sorted({0, 1, 2, 3, len(h) // 2, len(h), len(h) + 5, -1, -7})


def _check_family(pats, vocab, hists, subsets, kinds=(0, 1, 2)):
    brute = BruteStop(pats, vocab)
    images = [StopImage(image_bytes(pats, vocab, kind)) for kind in kinds]
    for S in subsets:
        for h in hists:
            for k in _news(h):
                want = brute(h, k, S)
                for kind, img in zip(kinds, images):   # every match kind gives one answer
                    assert img.stop(h, k, S) == want, (kind, h, k, S)
                if want is not None:
                    f = len(h) - min(max(k, 0), len(h))
                    assert want[1] >= f and 1 <= want[2] <= len(vocab[h[want[1]]])


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("seed", range(2))
def test_interpreter_equals_brute_force(name, seed):
    rng = np.random.default_rng(1000 * seed + CASES.index(name))
    pats, vocab, hists = _case(name, rng)
    subsets = [None, set(), {p for p in range(len(pats)) if rng.random() < 0.5}]
    _check_family(pats, vocab, hists, subsets)


@pytest.mark.parametrize("make", vf.WALKS + [lambda: vf.pieces(33), lambda: vf.pieces(100)],
                         ids=[w.__name__ for w in vf.WALKS] + ["pieces-33", "pieces-100"])
def test_interpreter_equals_brute_force_on_geometry_families(make):
    fam = make()
    _check_family(fam.patterns, fam.vocab, fam.histories, [None, {0}, set(range(1, len(fam.patterns)))], kinds=(0, 2))


def test_breaks_and_empty_entries_around_the_new_ids():
    pats = [b"abc", b"bc", b"ca"]
    vocab = [b"a", b"b", b"c", b"", b"ab", b"bca"]
    brute, img = BruteStop(pats, vocab), StopImage(image_bytes(pats, vocab))
    cases = [
        ([0, 1, 2], 1, (0, 2, 1, 3)),           # "abc" ends in the last id: the longest of abc / bc
        ([0, -1, 1, 2], 1, (1, 3, 1, 2)),       # a break before: only "bc"
        ([0, 1, -1, 2], 1, None),               # a break among the old ids cuts both
        ([0, 1, 2, -1], 2, (0, 2, 1, 3)),       # a break after the new id that holds the end
        ([0, 1, 2, -1], 1, None),               # ... which is not new when only the break is
        ([0] + [3] * 50 + [1] + [3] * 40 + [2], 1, (0, 92, 1, 3)),   # empty entries between the tail bytes
        ([4, 3, 3, 2], 3, (0, 3, 1, 3)),
        ([5], 1, (1, 0, 2, 2)),                 # "bc" ends at byte 1 of "bca", before "ca" at byte 2
        ([0, 1, 2], 0, None),                   # nothing is new
        ([0, 1, 2], 9, (0, 2, 1, 3)),           # more than the row: all of it is new
        ([], 1, None),
    ]
    for h, k, want in cases:
        assert brute(h, k) == want and img.stop(h, k) == want, (h, k)


def test_tie_rule_longest_then_lowest_pid():
    pats = [b"cd", b"bcd", b"bcd", b"d", b"xbcd"]
    vocab = [b"abcd", b"b", b"cd", b"xx"]
    brute, img = BruteStop(pats, vocab), StopImage(image_bytes(pats, vocab))
    for S, want in ((None, (1, 0, 4, 3)), ({2, 0, 3}, (2, 0, 4, 3)), ({0, 3}, (0, 0, 4, 2)), ({3}, (3, 0, 4, 1)), ({4}, None)):
        assert brute([0], 1, S) == want and img.stop([0], 1, S) == want, S
    # the earliest last byte wins over a longer match that ends later in the same id
    pats = [b"ab", b"abcdef"]
    vocab = [b"abcdef"]
    assert BruteStop(pats, vocab)([0]) == (0, 0, 2, 2) == StopImage(image_bytes(pats, vocab)).stop([0])


def test_long_pattern_over_one_byte_tokens():
    rng = np.random.default_rng(5)
    P = np.frombuffer(b"ab", dtype=np.uint8)[rng.integers(0, 2, 200)].tobytes()
    vocab = [b"a", b"b", b""]
    h = [b"ab".index(c) for c in P]
    pats = [P, b"q"]
    brute, img = BruteStop(pats, vocab), StopImage(image_bytes(pats, vocab))
    assert img.need == 199
    assert brute(h, 1) == img.stop(h, 1) == (0, 199, 1, 200)
    h2 = [0, 1] + h[:100] + [2] * 10 + h[100:]
    assert brute(h2, 1) == img.stop(h2, 1) == (0, len(h2) - 1, 1, 200)
    assert img.stop(h[:-1], 1) is None and img.stop([-1] + h[1:], 5) is None


def test_utf8_split_across_ids():
    pats = ["é".encode(), "naïve".encode()]
    vocab = [b"na", b"\xc3", b"\xaf", b"ve", b"\xa9"]
    brute, img = BruteStop(pats, vocab), StopImage(image_bytes(pats, vocab))
    assert brute([1, 4], 1) == img.stop([1, 4], 1) == (0, 1, 1, 2)
    assert brute([0, 1, 2, 3], 1) == img.stop([0, 1, 2, 3], 1) == (1, 3, 2, 6)


def test_no_patterns_and_need_zero():
    vocab = [b"a", b"", b"ab"]
    assert StopImage(image_bytes([], vocab)).stop([0, 2], 2) is None and BruteStop([], vocab)([0, 2], 2) is None
    img = StopImage(image_bytes([b"b"], vocab))
    assert img.need == 0
    assert img.stop([2, 0, 2], 1) == (0, 2, 2, 1) and img.stop([2, 0], 1) is None


@pytest.mark.parametrize("name", CASES)
def test_new_one_identity_with_completing_tokens(name):
    """new = 1: row h + [t] has a stop exactly when t completes a pattern after h (DESIGN §4.18's relation)."""
    rng = np.random.default_rng(77 + CASES.index(name))
    pats, vocab, hists = _case(name, rng)
    comp, img = BruteModel(pats, vocab), StopImage(image_bytes(pats, vocab))
    for S in (None, {p for p in range(len(pats)) if rng.random() < 0.5}):
        for h in hists[:10]:
            banned = set(comp(h, S))
            for t in range(len(vocab)):
                assert (img.stop(h + [t], 1, S) is not None) == (t in banned), (h, t, S)


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_export():
    assert "acb_vocab_stop" in _capi.EXPORTS and getattr(_capi.lib(), "acb_vocab_stop")


def _stop(L, h, **kw):
    img = np.zeros(16, dtype=np.uint8)
    tok = np.zeros(4, dtype=np.int64)
    off = np.array([0, 2], dtype=np.int64)
    out = np.zeros(4, dtype=np.int64)
    a = dict(a=h, img=img.ctypes.data, tok=tok.ctypes.data, tb=8, nt=4, off=off.ctypes.data, nr=1, k=1, news=None, out=out.ctypes.data,
             flt=None)
    a.update(kw)
    return L.acb_vocab_stop(a["a"], a["img"], a["tok"], a["tb"], a["nt"], a["off"], a["nr"], a["k"], a["news"], a["out"], a["flt"], None)


def test_stop_argument_errors_before_any_cuda_call():
    L, h = build_automaton([b"ab"])
    try:
        E = _capi.ACB_EINVAL
        for kw in (dict(a=None), dict(img=None), dict(tok=None), dict(off=None), dict(out=None), dict(tb=3), dict(tb=1), dict(tb=16),
                   dict(nt=1 << 60), dict(nr=-1), dict(nr=1 << 32), dict(k=-1), dict(k=-(1 << 63))):
            assert _stop(L, h, **kw) == E, kw
        assert "n_new" in (_stop(L, h, k=-1), _capi.last_error())[1]
        f = _capi.PatternFilter()
        f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = None, 1, None, 4
        assert _stop(L, h, flt=C.byref(f)) == E
        bits = np.zeros(1, dtype=np.uint32)
        f.dev_set_bits, f.n_sets = bits.ctypes.data, 0
        assert _stop(L, h, flt=C.byref(f)) == E
        f.n_sets, f.index_bytes = 1, 2
        assert _stop(L, h, flt=C.byref(f)) == E
    finally:
        L.acb_free(h)


# ---- Python argument errors that need no device --------------------------------------------------------------------------
def test_stop_argument_errors_without_a_device():
    v = BytesAhoCorasick([b"ab"]).vocabulary([b"a", b"b"])
    with pytest.raises(TypeError, match="tokens"):
        v.find_stop_device(torch.zeros(2, dtype=torch.int64), torch.tensor([0, 2]))
    with pytest.raises(TypeError, match="tokens"):
        v.find_stop_device([0, 1], torch.tensor([0, 2]))
    with pytest.raises(TypeError):
        v.find_stop([[0, 1], [1]])
    with pytest.raises(TypeError):
        v.find_stop([0.5, 1.0])
    with pytest.raises(ValueError, match="new"):
        v.find_stop([0, 1], new=-1)
    with pytest.raises(TypeError):
        v.find_stop([0, 1], new=1.5)
    with pytest.raises(TypeError):
        v.find_stop([0, 1], new="1")
    with pytest.raises(ValueError, match="new"):
        v.find_stop_batch([[0], [1]], new=[1])
    for bad in ([True, 1], [1.5, 1], np.array([[1], [1]]), 2.0, None):
        with pytest.raises(TypeError, match="new"):
            v.find_stop_batch([[0], [1]], new=bad)
    with pytest.raises(ValueError):
        v.find_stop_batch([[0], [1]], patterns=[[0]])
    assert v.find_stop_batch([]) == []


def test_host_counts_are_python_ints_of_any_size():
    """find_stop_batch's per-history counts keep their value: one beyond int64 still means the whole history."""
    from ahocorasick_rs_b200.matcher import _host_news
    assert _host_news([1 << 70, -3, np.int64(2)], 3) == [1 << 70, -3, 2]
    assert _host_news(torch.tensor([2, 0]), 2) == [2, 0]
    assert _host_news(np.uint8(3), 2) == [3, 3] and _host_news(torch.tensor(4), 1) == [4]
