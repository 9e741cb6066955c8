"""CPU tests of count_matches: the three C entry points refuse bad arguments before any CUDA call, the public methods
validate their arguments exactly as find_matches_as_indexes does and have no CPU fallback, and the two claims the count
kernels rest on hold against the oracle on thousands of seeded cases:
  - the non-overlapping count is the length of the chain NEXT(0), NEXT(end), ..., where NEXT(s) is what the serial
    selection picks once it restarts at s, and pointer jumping over (next, rank) pairs measures it;
  - the overlapping count of one haystack in windows that share max_pattern_len - 1 bytes is the sum of the windows'
    counts minus the counts of their shared heads."""
import bisect
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .spec_bruteforce import spec_find

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
KIND_NAMES = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def _automaton(kind=0):
    L = _capi.lib()
    pats = [b"hello", b"world"]
    offs = np.array([0, 5, 10], dtype=np.uint64)
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, 2, kind, -1, C.byref(h)) == 0
    return L, h


def _workspace(**null):
    ws = _capi.Workspace()
    for name, _ in _capi.Workspace._fields_:
        setattr(ws, name, 1 << 16 if "capacity" in name else FAKE)
    for name in null:
        setattr(ws, name, None)
    return ws


def _over(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, counts=FAKE, scratch=FAKE):
    return L.acb_count_overlapping(h, sieve, data, offs, n, total, counts, scratch, None)


def _non(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, plan=None, ws=None, counts=FAKE):
    if plan is None:
        plan = _capi.Plan()
        assert L.acb_plan_scan(h, FAKE if data is None else data, total, max(n, 0), C.byref(plan)) == 0
    return L.acb_count_non_overlapping(h, sieve, data, offs, n, total, C.byref(plan), C.byref(ws or _workspace()), counts, None)


def _rows(L, h, rows=FAKE, n=4, scratch=FAKE, count=FAKE):
    return L.acb_count_rows(h, rows, n, scratch, count, None)


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
        assert L.acb_count_overlapping(None, FAKE, FAKE, FAKE, 1, 16, FAKE, FAKE, None) == _capi.ACB_EINVAL
        non_cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(counts=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(ws=_workspace(dev_raw=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_total=1)), "workspace has a null buffer"),
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
        assert L.acb_count_non_overlapping(None, FAKE, FAKE, FAKE, 1, 16, C.byref(plan), C.byref(_workspace()), FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_count_non_overlapping(h, FAKE, FAKE, FAKE, 1, 16, None, C.byref(_workspace()), FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_count_non_overlapping(h, FAKE, FAKE, FAKE, 1, 16, C.byref(plan), None, FAKE, None) == _capi.ACB_EINVAL
        rows_cases = [
            (dict(rows=None), "null argument"),
            (dict(scratch=None), "null argument"),
            (dict(count=None), "null argument"),
            (dict(n=0xffffffff), "n_rows out of range"),
        ]
        for kw, msg in rows_cases:
            assert _rows(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert _rows(L, None) == _capi.ACB_EINVAL
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2], ids=KIND_NAMES[1:])
def test_overlapping_count_refuses_leftmost_kinds_before_any_cuda_call(kind):
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
        assert _rows(L, h) == _capi.ACB_ECUDA, _capi.last_error()
        assert _rows(L, h, rows=None, scratch=None, n=0) == _capi.ACB_ECUDA, _capi.last_error()
    finally:
        L.acb_free(h)


def _same_error(fn_a, fn_b):
    with pytest.raises(Exception) as a:
        fn_a()
    with pytest.raises(Exception) as b:
        fn_b()
    assert type(a.value) is type(b.value) and str(a.value) == str(b.value)
    return a.value


def test_count_matches_validates_like_find_matches_as_indexes():
    ac = AhoCorasick(["hello"])
    for bad in (b"hello", 12, None, ["hello"]):
        e = _same_error(lambda: ac.count_matches(bad), lambda: ac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            ac.count_matches_batch(["ok", bad])
    bac = BytesAhoCorasick([b"hello"])
    for bad in ("hello", 12, np.zeros((2, 2), dtype=np.uint8), np.arange(10, dtype=np.uint8)[::2]):
        e = _same_error(lambda: bac.count_matches(bad), lambda: bac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            bac.count_matches_batch([b"ok", bad])
    bad = np.arange(4, dtype=np.int32)   # not u8
    e = _same_error(lambda: bac.count_matches(bad), lambda: bac.find_matches_as_indexes(bad))
    assert isinstance(e, BufferError)
    for kind in (MatchKind.LeftmostFirst, MatchKind.LeftmostLongest):
        a, b = AhoCorasick(["a"], matchkind=kind), BytesAhoCorasick([b"a"], matchkind=kind)
        e = _same_error(lambda: a.count_matches("abc", overlapping=True), lambda: a.find_matches_as_indexes("abc", overlapping=True))
        assert isinstance(e, ValueError)
        e = _same_error(lambda: b.count_matches(b"abc", True), lambda: b.find_matches_as_indexes(b"abc", True))
        assert isinstance(e, ValueError)
        with pytest.raises(ValueError):
            a.count_matches_batch(["abc"], overlapping=True)
        with pytest.raises(ValueError):
            b.count_matches_device(None, None, overlapping=True)


def test_count_matches_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for kind in MatchKind:
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).count_matches("abc")
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).count_matches_batch(["abc", "x"])
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).count_matches(b"abc")
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).count_matches_device(torch.zeros(3, dtype=torch.uint8), torch.tensor([0, 3]))
    with pytest.raises(RuntimeError):
        AhoCorasick(["a"]).count_matches("abc", overlapping=True)


# ------------------------------------------------- the successor chain (what the count epilogue computes, in Python)
def next_selected(kind, recs, ends, s, max_len):
    """NEXT(s): the serial selection's inner loop, started at the first record whose end is after s."""
    lo = bisect.bisect_right(ends, s)
    if kind == 0:
        return next((j for j in range(lo, len(recs)) if recs[j][1] >= s), len(recs))
    best, at = None, len(recs)
    for j in range(lo, len(recs)):
        pid, st, en = recs[j]
        if best is not None and en > best[1] + max_len:
            break
        if st < s:
            continue
        if best is None or st < best[1]:
            better = True
        elif st == best[1]:
            better = (en > best[2] or (en == best[2] and pid < best[0])) if kind == 2 else pid < best[0]
        else:
            better = False
        if better:
            best, at = recs[j], j
    return at


def count_by_chain(kind, over, max_len):
    """The non-overlapping count from the overlapping list alone: successors, then pointer jumping over (next, rank)
    pairs in ceil(log2(n)) double-buffered rounds, then the rank of NEXT(0)."""
    recs = sorted(over, key=lambda m: (m[2], m[1], m[0]))   # the list order: end, start, pattern
    n = len(recs)
    if n == 0:
        return 0
    ends = [m[2] for m in recs]
    nxt = [next_selected(kind, recs, ends, m[2], max_len) for m in recs]
    assert all(j > i for i, j in enumerate(nxt))   # a successor always lies further on
    rank = [1] * n
    for _ in range(max(n - 1, 0).bit_length()):   # ceil(log2(n))
        nxt, rank = ([nxt[i] if nxt[i] == n else nxt[nxt[i]] for i in range(n)],
                     [rank[i] if nxt[i] == n else rank[i] + rank[nxt[i]] for i in range(n)])
    head = next_selected(kind, recs, ends, 0, max_len)
    return 0 if head == n else rank[head]


def _case(rng, case):
    alpha = b"abc" if case % 3 else b"ab"
    pats = [bytes(rng.choice(list(alpha), size=int(rng.integers(1, 6))).astype(np.uint8)) for _ in range(int(rng.integers(1, 9)))]
    if case % 5 == 0:
        pats.append(pats[int(rng.integers(0, len(pats)))])   # a duplicate
    if case % 7 == 0:
        pats.append(pats[0] + pats[-1])                      # nested patterns
    if case % 4 == 0:
        pats.append(b"a" * int(rng.integers(1, 4)))          # self-overlapping
    hay = bytes(rng.choice(list(alpha), size=int(rng.integers(0, 60))).astype(np.uint8))
    if case % 11 == 0:
        pats.append(hay + b"a")                              # longer than the haystack
    return pats, hay


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_successor_chain_counts_equal_the_oracles(kind):
    rng = np.random.default_rng(2000 + kind)
    nonzero = 0
    for case in range(3000):
        pats, hay = _case(rng, case)
        over = Oracle(pats, 0).find(hay, overlapping=True)
        want = len(Oracle(pats, kind).find(hay))
        assert count_by_chain(kind, over, max(len(p) for p in pats)) == want, (pats, hay)
        if case % 50 == 0:
            assert len(spec_find(pats, hay, KIND_NAMES[kind])) == want
        nonzero += want > 0
    assert nonzero > 1500


def test_window_heads_make_overlapping_counts_exact():
    rng = np.random.default_rng(77)
    for case in range(1500):
        pats, hay = _case(rng, case)
        max_len = max(len(p) for p in pats)
        halo = max_len - 1
        window = halo + int(rng.integers(1, 12))
        oracle = Oracle(pats, 0)
        total, w0 = 0, 0
        while True:
            w1 = min(w0 + window, len(hay))
            total += len(oracle.find(hay[w0:w1], overlapping=True))
            if w0 and halo:
                total -= len(oracle.find(hay[w0:w0 + halo], overlapping=True))
            if w1 >= len(hay):
                break
            w0 += window - halo
        assert total == len(oracle.find(hay, overlapping=True)), (pats, hay, window)
