"""GPU tests of the sieve (scan_sieve.cuh) at geometries the builder would not pick for these inputs (-m gpu): every
primary window W (1..8) against every ring depth R (1, 2, 4, 8 windows of text per warp), 16 KiB and 512-byte tasks,
code points, the filter budget (default, shallow: nothing on chip beyond the primary window, saturated: a 4 KiB
filter whose primary bitmap is nearly full), and reverse-trie nodes with 1, 8, 9, 255 and 256 children.  Every case
runs all five of the kernel's modes -- the match list (three kinds and overlapping), is_match, find_first, the counts
and the per-pattern counts -- and the two epilogues that read the ordered list for count_matches_by_pattern and
matching_patterns, against the CPU oracle, and asserts after every call that last_stats report the geometry it was
built for (a changed default that stops an input from reaching its corner fails here instead of passing silently)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import MatchKind, matcher  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, check_batch, dev, dev_at, make_ac  # noqa: E402
from .sieve_geometry_helpers import (assert_geometry, case_inputs, fanout, first_rows_of, geometry, hist_of, hits_of,  # noqa: E402
                                     hits_sums, host_geometry, planted)
from .sieve_inputs import FANOUTS, TWO_LEVEL  # noqa: E402

RINGS = (1, 2, 4, 8)
SHIFTS = (0, 1, 511)   # where the data starts after a 512-byte aligned address: moves the window and task grids
DEFAULT_TASK = 16384


def oracle(pats, kind, data, offs, overlapping=False, codepoints=False):
    return Oracle(pats, kind.name).scan_batch(data, offs, overlapping=overlapping, codepoints=codepoints)


def check_pattern_queries(ac, pats, d, o, want, counts, rec, overlapping=False):
    """count_matches_by_pattern and matching_patterns of one search against the oracle's records, with the geometry
    and the mode asserted after each call; the hits' row sums are the per-haystack counts and their column sums the
    per-pattern counts."""
    hist = ac.count_matches_by_pattern_device(d, o, overlapping).cpu().numpy()
    assert_geometry(ac, want)
    assert ac._ac.last_stats["mode"] == "pattern_counts"
    assert np.array_equal(hist, hist_of(rec, len(pats))), (ac._ac.matchkind, overlapping)
    got = [t.cpu().numpy() for t in ac.matching_patterns_device(d, o, overlapping)]
    assert_geometry(ac, want)
    assert ac._ac.last_stats["mode"] == "matching_patterns"
    for t, exp in zip(got, hits_of(rec, len(counts), len(pats))):
        assert np.array_equal(t, exp), (ac._ac.matchkind, overlapping)
    rows, cols = hits_sums(got, len(counts), len(pats))
    assert np.array_equal(rows, counts.astype(np.int64)) and np.array_equal(cols, hist)


def check_all_modes(pats, data, offs, want, codepoints=False, shift=0):
    """The four searches' lists, is_match, find_first for every kind, both counts, count_matches_by_pattern (the
    pattern mode for the overlapping search, the pattern epilogue for the others) and matching_patterns (the hits
    epilogue), each against the oracle, with the geometry asserted after every call.  -> overlapping matches in the
    batch."""
    d, o = dev_at(data, shift), dev(offs)
    over_total, over_counts, over_rec = oracle(pats, MatchKind.Standard, data, offs, overlapping=True)
    assert over_total > 0
    for kind in KINDS:
        ac = make_ac(pats, kind, codepoints)
        check_batch(pats, kind, data, offs, codepoints=codepoints, ac=ac, shift=shift)
        assert_geometry(ac, want)
        got = ac.find_first_device(d, o).cpu().numpy()
        assert_geometry(ac, want)
        assert np.array_equal(got, first_rows_of(*oracle(pats, kind, data, offs, codepoints=codepoints)[1:])), kind
        _, counts, rec = oracle(pats, kind, data, offs)
        got = ac.count_matches_device(d, o).cpu().numpy()
        assert_geometry(ac, want)
        assert np.array_equal(got, counts.astype(np.int64)), kind
        check_pattern_queries(ac, pats, d, o, want, counts, rec)
        if kind == MatchKind.Standard:
            check_batch(pats, kind, data, offs, overlapping=True, codepoints=codepoints, ac=ac, shift=shift)
            assert_geometry(ac, want)
            got = ac.count_matches_device(d, o, overlapping=True).cpu().numpy()
            assert_geometry(ac, want)
            assert np.array_equal(got, over_counts.astype(np.int64))
            got = ac.is_match_device(d, o).cpu().numpy()
            assert_geometry(ac, want)
            assert np.array_equal(got, over_counts > 0)
            check_pattern_queries(ac, pats, d, o, want, over_counts, over_rec, overlapping=True)
    return over_total


# ---------------------------------------------------------------- W x R, planted batch
@pytest.mark.parametrize("ring", RINGS)
@pytest.mark.parametrize("w", range(1, 9))
def test_window_by_ring(monkeypatch, w, ring):
    pats, data, offs = planted(False)
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_all_modes(pats, data, offs, {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, shift=SHIFTS[(w + ring) % 3])


@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("w", (1, 4, 5, 8))
def test_window_by_ring_small_tasks(monkeypatch, w, ring):
    """One window per task: every queue is drained at every task's end, every window starts a task."""
    pats, data, offs = planted(False)
    with geometry(monkeypatch, w, ring, 512):
        check_all_modes(pats, data, offs, {"window": w, "ring": ring, "task_bytes": 512}, shift=SHIFTS[(w + ring) % 3])


@pytest.mark.parametrize("ring", RINGS)
@pytest.mark.parametrize("w", (1, 3, 4, 5, 8))
def test_code_points_window_by_ring(monkeypatch, w, ring):
    """Multi-byte characters between and inside the occurrences: stage 1 takes each survivor's continuation count
    from the ring slot of its window."""
    pats, data, offs = planted(True)
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_all_modes(pats, data, offs, {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, codepoints=True,
                        shift=SHIFTS[(w + ring) % 3])


# ---------------------------------------------------------------- filter budget
BUDGET_W = 5
BUDGETS = {
    # name: (inputs, filter budget in bytes (None: what the default reserve leaves))
    "default": ("planted", None),
    "shallow": ("decoys", 8192),      # 1 000 more patterns in 8 KiB: the secondary filter holds the primary window only
    "saturated": ("dense", 4096),     # 100 000 patterns in the smallest budget: the primary bitmap nearly full
}


@pytest.mark.parametrize("utf8", [False, True], ids=["bytes", "utf8"])
@pytest.mark.parametrize("task_bytes", (DEFAULT_TASK, 512))
@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("budget", list(BUDGETS))
def test_filter_budget(monkeypatch, budget, ring, task_bytes, utf8):
    name, nbytes = BUDGETS[budget]
    case = (name, utf8)
    pats, data, offs = case_inputs(case)
    smem = matcher._Automaton._smem_optin(torch.cuda.current_device())
    host_budget = nbytes if nbytes is not None else max(4096, smem - matcher._Automaton.SIEVE_SMEM_RESERVE)
    W, last_level, probes, bloom_bytes, fill = host_geometry(case, host_budget, BUDGET_W)
    assert W == BUDGET_W
    if budget == "default":
        assert last_level == 16   # kSieveMaxLevel: the on-chip walk as deep as it goes
    elif budget == "shallow":
        assert last_level == W and fill < 0.05
    else:
        assert last_level == W and bloom_bytes == 4096 and fill >= 0.95, fill   # nearly every position reaches stage 1
    want = {"window": W, "last_level": last_level, "probes": probes, "bloom_bytes": bloom_bytes, "ring": ring,
            "task_bytes": task_bytes}
    with geometry(monkeypatch, BUDGET_W, ring, task_bytes, nbytes):
        check_all_modes(pats, data, offs, want, codepoints=utf8, shift=SHIFTS[(ring + task_bytes // 512) % 3])


# ---------------------------------------------------------------- reverse-trie fan-out
@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("w", (1, 5, 8))
@pytest.mark.parametrize("fan", list(FANOUTS) + [TWO_LEVEL])
def test_trie_fanout(monkeypatch, fan, w, ring):
    """A node with 1, 8 (the last linear scan), 9 (the first binary search), 255 or 256 children (a count that needs
    the ninth bit), children 0x00 and 0xff at the ends, and two levels of many children; the text puts each of the 256
    byte values before the core."""
    pats, data, offs = fanout(fan)
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_all_modes(pats, data, offs, {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, shift=SHIFTS[w % 3])
