"""Helpers shared by the sieve geometry tests and the pattern-set tests: the cached seeded inputs of
tests/sieve_inputs.py, forcing a sieve geometry (primary window, ring depth, task size, filter budget) and asserting it,
the skip counters the task grid predicts for is_match and find_first, `subset_scan_batch`, the CPU reference of a
batch in which every haystack searches for its own subset of the patterns, and the references of
count_matches_by_pattern and matching_patterns taken from the oracle's records."""
import contextlib
import functools

import numpy as np

from ahocorasick_rs_b200 import MatchKind, _capi, matcher
from oracle import Oracle

from .sieve_inputs import dense_case, fanout_case, planted_case
from .sieve_interp import SieveImage


@functools.lru_cache(maxsize=None)
def planted(utf8, decoys=0):
    return planted_case(utf8, decoys=decoys)


@functools.lru_cache(maxsize=None)
def dense(utf8):
    return dense_case(utf8)


@functools.lru_cache(maxsize=None)
def fanout(f):
    return fanout_case(f)


def case_inputs(case):
    name, utf8 = case
    if name == "dense":
        return dense(utf8)
    return planted(utf8, 1000 if name == "decoys" else 0)


@functools.lru_cache(maxsize=None)
def host_geometry(case, budget, w):
    """What the builder makes of a case at a filter budget, on the host (tests/sieve_interp.SieveImage: the same C
    builder) -> (window, last_level, probes, bloom_bytes, primary bitmap fill)."""
    pats = case_inputs(case)[0]
    img = SieveImage(pats, 0, budget, w)
    fill = float(np.unpackbits(img.bloom[:img.prim_words].view(np.uint8)).mean())
    return img.W, img.last_level, img.n_probes, img.bloom_words * 4, fill


@contextlib.contextmanager
def geometry(monkeypatch, w, ring, task_bytes, budget=None):
    """Sieve scans on this thread with primary window w (automata built inside: the image is built at the first
    scan), ring depth `ring`, tasks of task_bytes and, when given, filters built for `budget` bytes."""
    import torch
    monkeypatch.setattr(matcher._Automaton, "SIEVE_W_MAX", w)
    if budget is not None:
        smem = matcher._Automaton._smem_optin(torch.cuda.current_device())
        monkeypatch.setattr(matcher._Automaton, "SIEVE_SMEM_RESERVE", smem - budget)
    _capi.set_tuning(5, 0, task_bytes, 0, sieve_ring=ring)
    try:
        yield
    finally:
        _capi.set_tuning(0)


def assert_geometry(ac, want):
    st = ac._ac.last_stats
    assert st["engine"] == "sieve", st
    for k, v in want.items():
        assert st[k] == v, (k, v, st)


# ---------------------------------------------------------------- skip counters the task grid predicts
def predicted_any_skips(ptr, offs, flags, T):
    """is_match: tasks skipped whole and windows not scanned, from the task grid (see acb_any_match in
    include/acb200.h), for flags that do not change during the call."""
    origin = -(ptr & 511)
    total = int(offs[-1])
    n_tasks = (total - origin + T - 1) // T
    tasks = windows = 0
    for k in range(n_tasks):
        t_lo = origin + k * T
        lo, hi = max(t_lo, 0), min(t_lo + T, total)
        if lo >= hi:
            continue
        tail = int(np.searchsorted(offs, hi - 1, side="right")) - 1
        if not flags[tail]:
            continue
        tail_s = int(offs[tail]) - t_lo
        lo_r, hi_r = lo - t_lo, hi - t_lo
        if tail_s <= lo_r:
            tasks += 1
            continue
        wfirst, wlast = lo_r & ~511, (hi_r - 1) & ~511
        for w in range(wfirst + 512, wlast + 1, 512):
            if w >= tail_s:
                windows += (wlast - w) // 512 + 1
                break
    return tasks, windows


def predicted_first_skips(ptr, offs, key_hi, T, kind, max_len):
    """find_first: tasks skipped whole and windows not scanned, from the task grid (see acb_find_first in
    include/acb200.h), for keys that do not change during the call (key_hi: the high words, 0xffffffff where there is
    no match)."""
    origin = -(ptr & 511)
    total = int(offs[-1])
    n_tasks = (total - origin + T - 1) // T
    tasks = windows = 0
    for k in range(n_tasks):
        t_lo = origin + k * T
        lo, hi = max(t_lo, 0), min(t_lo + T, total)
        if lo >= hi:
            continue
        tail = int(np.searchsorted(offs, hi - 1, side="right")) - 1
        tail_s = int(offs[tail]) - t_lo
        lo_r, hi_r = lo - t_lo, hi - t_lo

        def cannot_win(rel):
            e = rel - tail_s + 1
            return (e if kind == MatchKind.Standard else max(e - max_len, 0)) > int(key_hi[tail])

        if tail_s <= lo_r and cannot_win(lo_r):
            tasks += 1
            continue
        wfirst, wlast = lo_r & ~511, (hi_r - 1) & ~511
        for w in range(wfirst + 512, wlast + 1, 512):
            if w >= tail_s and cannot_win(w):
                windows += (wlast - w) // 512 + 1
                break
    return tasks, windows


# ---------------------------------------------------------------- the pattern-set reference
def subset_scan_batch(pats, kind, data, offs, sets, set_index, overlapping=False, codepoints=False):
    """The CPU oracle's answer for a batch whose haystack h searches only for the patterns of sets[set_index[h]] ->
    (total, counts, records) in the format of Oracle.scan_batch.  The haystacks are grouped by set, each group is scanned
    by an oracle built from that set's patterns (in their original relative order), and the pattern ids and haystack
    numbers are mapped back to the full automaton and the batch.  An index outside [0, len(sets)) admits nothing."""
    kname = getattr(kind, "name", kind)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offs = np.asarray(offs, dtype=np.int64)
    idx = np.asarray(set_index, dtype=np.int64)
    n = len(offs) - 1
    counts = np.zeros(n, dtype=np.uint32)
    parts = [np.zeros((0, 4), dtype=np.uint32)]
    for g in np.unique(idx).tolist():
        ids = sorted({int(p) for p in sets[g]}) if 0 <= g < len(sets) else []
        if not ids:
            continue
        hs = np.flatnonzero(idx == g)
        goffs = np.zeros(len(hs) + 1, dtype=np.int64)
        np.cumsum(offs[hs + 1] - offs[hs], out=goffs[1:])
        gdata = np.concatenate([data[offs[h]:offs[h + 1]] for h in hs] + [np.zeros(0, dtype=np.uint8)])
        _, c, rec = Oracle([pats[i] for i in ids], kname).scan_batch(gdata, goffs, overlapping=overlapping, codepoints=codepoints)
        counts[hs] = c
        rec = rec.copy()
        rec[:, 0] = hs[rec[:, 0]]
        rec[:, 1] = np.asarray(ids, dtype=np.uint32)[rec[:, 1]]
        parts.append(rec)
    rec = np.concatenate(parts)
    rec = rec[np.argsort(rec[:, 0], kind="stable")]
    return int(counts.sum()), counts, rec


def first_rows_of(counts, rec):
    """A batch's first record per haystack from (counts, records) -> (n, 3) int64 rows, -1 where there is none."""
    rows = np.full((len(counts), 3), -1, dtype=np.int64)
    at = np.concatenate([[0], np.cumsum(counts.astype(np.int64))[:-1]])
    has = counts > 0
    rows[has] = rec[at[has]][:, 1:4].astype(np.int64)
    return rows


# ---------------------------------------------------------------- count_matches_by_pattern and matching_patterns
def hist_of(rec, n_patterns):
    """count_matches_by_pattern from a batch's records -> int64 (n_patterns,): the bincount of the pattern column."""
    return np.bincount(rec[:, 1].astype(np.int64), minlength=n_patterns)


def hits_of(rec, n_haystacks, n_patterns):
    """matching_patterns from a batch's records -> (row_offsets, patterns, counts) as int64 numpy arrays: each
    haystack's distinct pattern ids, ascending, and how many of its records have each."""
    keys, counts = np.unique(rec[:, 0].astype(np.int64) * n_patterns + rec[:, 1].astype(np.int64), return_counts=True)
    row_offsets = np.searchsorted(keys, np.arange(n_haystacks + 1, dtype=np.int64) * n_patterns)
    return row_offsets.astype(np.int64), keys % n_patterns, counts.astype(np.int64)


def oracle_hist(pats, data, offs, kind, overlapping):
    _, _, rec = Oracle(pats, kind.value).scan_batch(data, offs, overlapping=overlapping)
    return hist_of(rec, len(pats))


def oracle_hits(pats, data, offs, kind, overlapping):
    """-> (row_offsets, patterns, counts) as int64 numpy arrays, from the oracle's records."""
    _, _, rec = Oracle(pats, kind.value).scan_batch(data, offs, overlapping=overlapping)
    return hits_of(rec, len(offs) - 1, len(pats))


def hits_sums(hits, n_haystacks, n_patterns):
    """The row sums (per haystack) and column sums (per pattern) of a hits triple -> two int64 arrays."""
    ro, p, c = (np.asarray(t, dtype=np.int64) for t in hits)
    rows = np.zeros(n_haystacks, dtype=np.int64)
    np.add.at(rows, np.repeat(np.arange(n_haystacks), np.diff(ro)), c)
    cols = np.zeros(n_patterns, dtype=np.int64)
    np.add.at(cols, p, c)
    return rows, cols
