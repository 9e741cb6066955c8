"""CPU tests of count_matches_by_pattern: the two C entry points refuse bad arguments before any CUDA call, the public
methods validate their arguments exactly as count_matches does and have no CPU fallback, and the two claims the
pattern kernels rest on hold against the oracle on thousands of seeded cases:
  - marking the chain while pointer jumping (mark NEXT(0); in round k every marked record marks its round-k successor)
    marks exactly the non-overlapping selection, whatever order the records of a round run in and whether a mark set
    earlier in the same round is seen;
  - the overlapping per-pattern counts of one haystack in windows that share max_pattern_len - 1 bytes are the windows'
    histograms minus the histograms of their shared heads."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .test_count_cpu import FAKE, KIND_NAMES, _automaton, _case, _same_error, _workspace, next_selected


def _over(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, counts=FAKE, scratch=FAKE):
    return L.acb_pattern_counts_overlapping(h, sieve, data, offs, n, total, counts, scratch, None)


def _non(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, plan=None, ws=None, counts=FAKE):
    if plan is None:
        plan = _capi.Plan()
        assert L.acb_plan_scan(h, FAKE if data is None else data, total, max(n, 0), C.byref(plan)) == 0
    return L.acb_pattern_counts_non_overlapping(h, sieve, data, offs, n, total, C.byref(plan), C.byref(ws or _workspace()), counts, None)


def test_entry_points_reject_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        over_cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(counts=None), "null argument"),
            (dict(scratch=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31"),
            ({}, "acb_sieve_build has not been called"),   # valid arguments, but no sieve image yet
        ]
        for kw, msg in over_cases:
            assert _over(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_pattern_counts_overlapping(None, FAKE, FAKE, FAKE, 1, 16, FAKE, FAKE, None) == _capi.ACB_EINVAL
        non_cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(counts=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(ws=_workspace(dev_raw=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_raw_seq=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_match_offsets=1)), "workspace has a null buffer"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31"),
            (dict(plan=_capi.Plan()), "plan does not match"),
            ({}, "acb_sieve_build has not been called"),
        ]
        for kw, msg in non_cases:
            assert _non(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        plan = _capi.Plan()
        assert L.acb_pattern_counts_non_overlapping(None, FAKE, FAKE, FAKE, 1, 16, C.byref(plan), C.byref(_workspace()), FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_pattern_counts_non_overlapping(h, FAKE, FAKE, FAKE, 1, 16, None, C.byref(_workspace()), FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_pattern_counts_non_overlapping(h, FAKE, FAKE, FAKE, 1, 16, C.byref(plan), None, FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2], ids=KIND_NAMES[1:])
def test_overlapping_pattern_counts_refuse_leftmost_kinds_before_any_cuda_call(kind):
    L, h = _automaton(kind)
    try:
        launches = L.acb_launch_count()
        assert _over(L, h) == _capi.ACB_EUNSUPPORTED            # (no sieve image yet: refused before that check too)
        assert "does not support overlapping searches" in _capi.last_error()
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        assert _over(L, h) == _capi.ACB_EUNSUPPORTED
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_entry_points_need_a_device_past_the_checks(kind):
    """Past the argument checks the calls need CUDA: without a device they fail with ACB_ECUDA, never a CPU answer."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the pointers here are not device memory")
    L, h = _automaton(kind)
    try:
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        for total, data in ((16, FAKE), (0, None)):
            if kind == 0:
                assert _over(L, h, data=data, total=total) == _capi.ACB_ECUDA, _capi.last_error()
            assert _non(L, h, data=data, total=total) == _capi.ACB_ECUDA, _capi.last_error()
    finally:
        L.acb_free(h)


def test_count_matches_by_pattern_validates_like_count_matches():
    ac = AhoCorasick(["hello"])
    for bad in (b"hello", 12, None, ["hello"]):
        e = _same_error(lambda: ac.count_matches_by_pattern(bad), lambda: ac.count_matches(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            ac.count_matches_by_pattern_batch(["ok", bad])
    bac = BytesAhoCorasick([b"hello"])
    for bad in ("hello", 12, np.zeros((2, 2), dtype=np.uint8), np.arange(10, dtype=np.uint8)[::2]):
        e = _same_error(lambda: bac.count_matches_by_pattern(bad), lambda: bac.count_matches(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            bac.count_matches_by_pattern_batch([b"ok", bad])
    bad = np.arange(4, dtype=np.int32)   # not u8
    e = _same_error(lambda: bac.count_matches_by_pattern(bad), lambda: bac.count_matches(bad))
    assert isinstance(e, BufferError)
    for kind in (MatchKind.LeftmostFirst, MatchKind.LeftmostLongest):
        a, b = AhoCorasick(["a"], matchkind=kind), BytesAhoCorasick([b"a"], matchkind=kind)
        e = _same_error(lambda: a.count_matches_by_pattern("abc", overlapping=True), lambda: a.count_matches("abc", overlapping=True))
        assert isinstance(e, ValueError)
        e = _same_error(lambda: b.count_matches_by_pattern(b"abc", True), lambda: b.count_matches(b"abc", True))
        assert isinstance(e, ValueError)
        with pytest.raises(ValueError):
            a.count_matches_by_pattern_batch(["abc"], overlapping=True)
        with pytest.raises(ValueError):
            b.count_matches_by_pattern_device(None, None, overlapping=True)


def test_count_matches_by_pattern_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for kind in MatchKind:
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).count_matches_by_pattern("abc")
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).count_matches_by_pattern_batch(["abc", "x"])
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).count_matches_by_pattern(b"abc")
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).count_matches_by_pattern_device(torch.zeros(3, dtype=torch.uint8), torch.tensor([0, 3]))
    with pytest.raises(RuntimeError):
        AhoCorasick(["a"]).count_matches_by_pattern("abc", overlapping=True)


# ------------------------------------------------- the marked chain (what the pattern epilogue computes, in Python)
def marked_by_jumping(kind, over, max_len, rng):
    """The selection from the overlapping list alone: successors, mark[NEXT(0)], then ceil(log2(n)) double-buffered rounds
    of pointer jumping in which every marked record marks its round's successor.  Inside a round the records run in a
    random order, and each one reads the marks as they are at that moment (marks set earlier in the round included)."""
    recs = sorted(over, key=lambda m: (m[2], m[1], m[0]))   # the list order: end, start, pattern
    n = len(recs)
    if n == 0:
        return []
    ends = [m[2] for m in recs]
    nxt = [next_selected(kind, recs, ends, m[2], max_len) for m in recs]
    mark = [False] * n
    head = next_selected(kind, recs, ends, 0, max_len)
    if head < n:
        mark[head] = True
    for _ in range(max(n - 1, 0).bit_length()):   # ceil(log2(n))
        new = list(nxt)
        for i in rng.permutation(n):
            j = nxt[i]
            if j < n:
                if mark[i]:
                    mark[j] = True
                new[i] = nxt[j]
        nxt = new
    return [recs[i] for i in range(n) if mark[i]]


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_marked_chain_is_the_oracles_selection(kind):
    rng = np.random.default_rng(4000 + kind)
    nonzero = 0
    for case in range(3000):
        pats, hay = _case(rng, case)
        over = Oracle(pats, 0).find(hay, overlapping=True)
        want = Oracle(pats, kind).find(hay)
        got = marked_by_jumping(kind, over, max(len(p) for p in pats), rng)
        assert sorted(got) == sorted(tuple(m) for m in want), (pats, hay)
        nonzero += len(want) > 0
    assert nonzero > 1500


def _hist(oracle, hay, n_patterns):
    found = oracle.find(hay, overlapping=True)
    return np.bincount(np.array([m[0] for m in found], dtype=np.int64), minlength=n_patterns)


def test_window_heads_make_overlapping_pattern_counts_exact():
    rng = np.random.default_rng(78)
    for case in range(1500):
        pats, hay = _case(rng, case)
        max_len = max(len(p) for p in pats)
        halo = max_len - 1
        window = halo + int(rng.integers(1, 12))
        oracle = Oracle(pats, 0)
        total, w0 = np.zeros(len(pats), dtype=np.int64), 0
        while True:
            w1 = min(w0 + window, len(hay))
            total += _hist(oracle, hay[w0:w1], len(pats))
            if w0 and halo:
                total -= _hist(oracle, hay[w0:w0 + halo], len(pats))
            if w1 >= len(hay):
                break
            w0 += window - halo
        assert np.array_equal(total, _hist(oracle, hay, len(pats))), (pats, hay, window)
