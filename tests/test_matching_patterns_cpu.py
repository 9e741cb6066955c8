"""CPU tests of matching_patterns: acb_pattern_hits refuses bad arguments before any CUDA call (and overlapping searches
on leftmost automata with ACB_EUNSUPPORTED), the public methods validate their arguments exactly as count_matches does
and have no CPU fallback, and a Python model of the hits epilogue equals Counter of the oracle's records on thousands
of seeded batches of every kind and the overlapping search.  The model follows the kernel step by step, with the long
stretch limit and the counter-row tile patched small so that every path runs: short stretches sorted by the warp's
register network or by the flip-form network over a buffer and run-length encoded, long stretches aggregated in counter
rows and compacted by tile prefixes, every haystack's hits staged at its stretch offset, then offsets and packing."""
import bisect
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .test_count_cpu import FAKE, KIND_NAMES, _automaton, _case, _same_error, _workspace, next_selected
from .test_pattern_counts_cpu import marked_by_jumping


def _hits(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, overlapping=0, plan=None, ws=None, rows=FAKE, words=64):
    if plan is None:
        plan = _capi.Plan()
        assert L.acb_plan_scan(h, FAKE if data is None else data, total, max(n, 0), C.byref(plan)) == 0
    return L.acb_pattern_hits(h, sieve, data, offs, n, total, overlapping, C.byref(plan), C.byref(ws or _workspace()), rows, words, None)


def test_entry_point_rejects_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(rows=None), "null argument"),
            (dict(rows=FAKE + 4), "dev_rows must be 8-byte aligned"),
            (dict(overlapping=2), "overlapping must be 0 or 1"),
            (dict(ws=_workspace(dev_raw=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_raw_seq=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_out=1)), "workspace has a null buffer"),
            (dict(ws=_workspace(dev_match_offsets=1)), "workspace has a null buffer"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31"),
            (dict(plan=_capi.Plan()), "plan does not match"),
            ({}, "acb_sieve_build has not been called"),   # valid arguments, but no sieve image yet
            (dict(rows=None, words=0), "acb_sieve_build has not been called"),   # (no rows at all is valid)
        ]
        for kw, msg in cases:
            assert _hits(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        plan = _capi.Plan()
        assert L.acb_pattern_hits(None, FAKE, FAKE, FAKE, 1, 16, 0, C.byref(plan), C.byref(_workspace()), FAKE, 64, None) == _capi.ACB_EINVAL
        assert L.acb_pattern_hits(h, FAKE, FAKE, FAKE, 1, 16, 0, None, C.byref(_workspace()), FAKE, 64, None) == _capi.ACB_EINVAL
        assert L.acb_pattern_hits(h, FAKE, FAKE, FAKE, 1, 16, 0, C.byref(plan), None, FAKE, 64, None) == _capi.ACB_EINVAL
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2], ids=KIND_NAMES[1:])
def test_overlapping_hits_refuse_leftmost_kinds_before_any_cuda_call(kind):
    L, h = _automaton(kind)
    try:
        launches = L.acb_launch_count()
        assert _hits(L, h, overlapping=1) == _capi.ACB_EUNSUPPORTED   # (no sieve image yet: refused before that check too)
        assert "does not support overlapping searches" in _capi.last_error()
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        assert _hits(L, h, overlapping=1) == _capi.ACB_EUNSUPPORTED
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_entry_point_needs_a_device_past_the_checks(kind):
    """Past the argument checks the call needs CUDA: without a device it fails with ACB_ECUDA, never a CPU answer."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the pointers here are not device memory")
    L, h = _automaton(kind)
    try:
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        for total, data in ((16, FAKE), (0, None)):
            for overlapping in ([0, 1] if kind == 0 else [0]):
                assert _hits(L, h, data=data, total=total, overlapping=overlapping) == _capi.ACB_ECUDA, _capi.last_error()
            assert _hits(L, h, data=data, total=total, rows=None, words=0) == _capi.ACB_ECUDA, _capi.last_error()
    finally:
        L.acb_free(h)


def test_row_words_follow_the_layout():
    # n_patterns counters padded to even, then u64 [haystack, one word per 2048 counters]
    L = _capi.lib()
    for p, want in ((1, 2 + 2 + 2), (2, 2 + 2 + 2), (3, 4 + 2 + 2), (2048, 2048 + 2 + 2), (2049, 2050 + 2 + 4),
                    (100_000, 100_000 + 2 + 2 * 49)):
        assert L.acb_pattern_hit_row_words(p) == _row_words(p) == want


def test_matching_patterns_validates_like_count_matches():
    ac = AhoCorasick(["hello"])
    for bad in (b"hello", 12, None, ["hello"]):
        e = _same_error(lambda: ac.matching_patterns(bad), lambda: ac.count_matches(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            ac.matching_patterns_batch(["ok", bad])
    bac = BytesAhoCorasick([b"hello"])
    for bad in ("hello", 12, np.zeros((2, 2), dtype=np.uint8), np.arange(10, dtype=np.uint8)[::2]):
        e = _same_error(lambda: bac.matching_patterns(bad), lambda: bac.count_matches(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            bac.matching_patterns_batch([b"ok", bad])
    bad = np.arange(4, dtype=np.int32)   # not u8
    e = _same_error(lambda: bac.matching_patterns(bad), lambda: bac.count_matches(bad))
    assert isinstance(e, BufferError)
    for kind in (MatchKind.LeftmostFirst, MatchKind.LeftmostLongest):
        a, b = AhoCorasick(["a"], matchkind=kind), BytesAhoCorasick([b"a"], matchkind=kind)
        e = _same_error(lambda: a.matching_patterns("abc", overlapping=True), lambda: a.count_matches("abc", overlapping=True))
        assert isinstance(e, ValueError)
        e = _same_error(lambda: b.matching_patterns(b"abc", True), lambda: b.count_matches(b"abc", True))
        assert isinstance(e, ValueError)
        with pytest.raises(ValueError):
            a.matching_patterns_batch(["abc"], overlapping=True)
        with pytest.raises(ValueError):
            b.matching_patterns_device(None, None, overlapping=True)
        with pytest.raises(ValueError):
            a.matching_patterns_device(None, None, overlapping=True)


def test_matching_patterns_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for kind in MatchKind:
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).matching_patterns("abc")
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).matching_patterns_batch(["abc", "x"])
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).matching_patterns(b"abc")
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).matching_patterns_device(torch.zeros(3, dtype=torch.uint8), torch.tensor([0, 3]))
    with pytest.raises(RuntimeError):
        AhoCorasick(["a"]).matching_patterns("abc", overlapping=True)


# ------------------------------------------------- the hits epilogue, in Python
def _row_words(p, tile=2048):
    return (p + 1) // 2 * 2 + 2 + 2 * ((p + tile - 1) // tile)


def warp_sort32(keys):
    """The register network: lane l holds keys[l]; partners by xor, direction by bit k of the lane."""
    x = list(keys)
    k = 2
    while k <= 32:
        j = k >> 1
        while j:
            y = [x[lane ^ j] for lane in range(32)]
            x = [min(x[l], y[l]) if ((l & j) == 0) == ((l & k) == 0) else max(x[l], y[l]) for l in range(32)]
            j >>= 1
        k <<= 1
    return x


def warp_sort_keys(keys):
    """The flip-form network over keys[0 .. n): every comparator puts the smaller key first; partners past n skipped."""
    n = len(keys)
    half = (1 << (n - 1).bit_length()) >> 1 if n > 1 else 0
    k = 2
    while k <= 2 * half:
        j = k >> 1
        while j:
            for p in range(half):
                a = ((p & ~(j - 1)) << 1) | (p & (j - 1))
                b = a ^ (k - 1) if j == k >> 1 else a ^ j
                if b < n and keys[a] > keys[b]:
                    keys[a], keys[b] = keys[b], keys[a]
            j >>= 1
        k <<= 1
    return keys


def runs(keys, h):
    """Run-length encoding of sorted keys, each run's end found by binary search as warp_runs does."""
    out = []
    for j, k in enumerate(keys):
        if j == 0 or keys[j - 1] != k:
            end = bisect.bisect_right(keys, k, j + 1)
            out.append((h, k, end - j))
    return out


def hits_model(kind, overlapping, hays, pats, rng, long_limit, smem_keys, tile):
    """acb_pattern_hits in Python, up to the staging: -> (d_h per haystack, the staged hits (haystack, pattern, count)
    at each haystack's stretch offset in the ordered list, which paths ran)."""
    P, max_len = len(pats), max(len(p) for p in pats)
    over = Oracle(pats, 0)
    # phases 1-3: the ordered overlapping list, haystack by haystack (end, start, pattern)
    ordered = []
    for h, hay in enumerate(hays):
        ordered += [(h, pid, s, e) for pid, s, e in sorted(over.find(hay, overlapping=True), key=lambda m: (m[2], m[1], m[0]))]
    staged = [None] * len(ordered)
    d = [0] * len(hays)
    paths = Counter()
    rows = []
    i = 0
    while i < len(ordered):
        h = ordered[i][0]
        a = i
        while a < len(ordered) and ordered[a][0] == h:
            a += 1
        stretch = [(pid, s, e) for _, pid, s, e in ordered[i:a]]
        if len(stretch) <= long_limit:
            if overlapping:
                sel = stretch
            else:   # the serial selection: the chain NEXT(0), NEXT(end), ...
                ends = [m[2] for m in stretch]
                sel, j = [], next_selected(kind, stretch, ends, 0, max_len)
                while j < len(stretch):
                    sel.append(stretch[j])
                    j = next_selected(kind, stretch, ends, stretch[j][2], max_len)
            pids = [m[0] for m in sel]
            if len(pids) <= 32:
                paths["registers"] += 1
                srt = warp_sort32(pids + [0xffffffff] * (32 - len(pids)))[:len(pids)]
            else:
                paths["shared" if len(pids) <= smem_keys else "slice"] += 1
                srt = warp_sort_keys(list(pids))
            hs = runs(srt, h)
        else:
            paths["row"] += 1
            sel = stretch if overlapping else marked_by_jumping(kind, stretch, max_len, rng)
            row = [0] * P
            for pid, _, _ in sel:
                row[pid] += 1
            rows.append(row)
            # tile sums, then each tile's start within the row: the nonzero counters in pid order
            tiles = [sum(1 for c in row[t:t + tile] if c) for t in range(0, P, tile)]
            hs = []
            for t in range(len(tiles)):
                at = sum(tiles[:t])
                for p in range(t * tile, min(P, (t + 1) * tile)):
                    if row[p]:
                        assert len(hs) == at
                        hs.append((h, p, row[p]))
                        at += 1
        assert len(hs) <= a - i   # the staged slices never overlap
        staged[i:i + len(hs)] = hs   # at the stretch's offset
        d[h] = len(hs)
        i = a
    return d, staged, paths


@pytest.mark.parametrize("search", [(0, False), (0, True), (1, False), (2, False)],
                         ids=["Standard", "Standard-overlapping", "LeftmostFirst", "LeftmostLongest"])
def test_hits_model_equals_counter_of_the_oracles_records(search):
    kind, overlapping = search
    rng = np.random.default_rng(5000 + 2 * kind + overlapping)
    paths = Counter()
    for case in range(1200):
        pats, _ = _case(rng, case)
        hays = [_case(rng, case + 7 * k)[1] * int(rng.integers(1, 4)) for k in range(int(rng.integers(1, 6)))]
        if case % 9 == 0:
            hays.append(b"")
        long_limit = int(rng.integers(2, 80))
        smem_keys = int(rng.integers(33, 64))
        tile = int(rng.integers(1, 4))
        d, staged, p = hits_model(kind, overlapping, hays, pats, rng, long_limit, smem_keys, tile)
        paths += p
        # phases 5-6 and the pack: output o belongs to the last haystack whose offset is <= o
        offs = np.concatenate([[0], np.cumsum(d)]).astype(np.int64)
        starts, i = {}, 0
        ordered_lens = [len(Oracle(pats, 0).find(hay, overlapping=True)) for hay in hays]
        for h, ln in enumerate(ordered_lens):
            starts[h] = i
            i += ln
        out = []
        for o in range(int(offs[-1])):
            h = int(np.searchsorted(offs, o, side="right")) - 1
            out.append(staged[starts[h] + o - int(offs[h])])
        want = []
        for h, hay in enumerate(hays):
            c = Counter(m[0] for m in Oracle(pats, kind).find(hay, overlapping=overlapping))
            want += [(h, pid, c[pid]) for pid in sorted(c)]
        assert out == want, (pats, hays, long_limit)
    assert all(paths[k] >= 10 for k in ("registers", "shared", "slice", "row")), paths
