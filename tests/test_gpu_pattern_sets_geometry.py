"""GPU tests of pattern sets (DESIGN 4.13: sieve_scan_filtered_kernel, first_rows_filtered_kernel, the filtered stream
resolve) at every sieve geometry test_gpu_sieve_geometry.py runs, at the filter's edges and through its early exits
(-m gpu).  Each input gets a small family of sets built for a corner of the filter -- empty, all, shallow-only (a longer
pattern not admitted where a shorter one is), the later copy of a duplicate, the long pattern, word-edge pids, a core
without its trie children and the reverse -- and the host asserts, from the full overlapping oracle rows, that each set
reaches what it was built for and that filtering the unfiltered result afterwards would be wrong for it (or, for the
few sets no unadmitted match can hide anything from, that it would be right: those are listed).  Every device
answer is compared with `subset_scan_batch` (the oracle of each haystack's subset, ids mapped back)."""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, TokenAhoCorasick, matcher  # noqa: E402
from ahocorasick_rs_b200.matcher import PatternSets  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, dev, dev_at, forced, make_ac  # noqa: E402
from .sieve_geometry_helpers import (assert_geometry, case_inputs, fanout, first_rows_of, geometry, host_geometry,  # noqa: E402
                                     predicted_any_skips, predicted_first_skips, subset_scan_batch)
from .sieve_inputs import FANOUTS, PAT_LENGTHS, TWO_LEVEL  # noqa: E402

RINGS = (1, 2, 4, 8)
SHIFTS = (0, 1, 511)   # where the data starts after a 512-byte aligned address: moves the window and task grids
DEFAULT_TASK = 16384

# pids of the planted case (tests/sieve_inputs.planted_case)
_N = len(PAT_LENGTHS)
P24 = PAT_LENGTHS.index(24)
P16 = PAT_LENGTHS.index(16)
SUFFIX9, SUFFIX12 = _N, _N + 1           # p24[-9:], p24[-12:]: nested suffixes of the 24-byte pattern
Q8, Q11, P16_DUP, Q8_DUP = _N + 4, _N + 5, _N + 6, _N + 7
LONG = _N + 8                            # 600 bytes: longer than a window


def inputs(case):
    return fanout(case[1]) if case[0] == "fanout" else case_inputs(case)


def word_edges(P):
    """pids at bit 0 and bit 31 of their word, and the last pid when it ends a partial word"""
    return sorted({p for p in range(P) if p % 32 in (0, 31)} | ({P - 1} if P % 32 else set()))


@functools.lru_cache(maxsize=None)
def overlapping_rows(case):
    pats, data, offs = inputs(case)
    return Oracle(pats, "Standard").scan_batch(data, offs, overlapping=True)[2]


@functools.lru_cache(maxsize=None)
def family(case):
    """-> (names, sets, exact_after): the case's pattern sets, and the names of those for which filtering the
    unfiltered result afterwards happens to give the right answer (no admitted match can be hidden)."""
    pats, _, _ = inputs(case)
    P = len(pats)
    rec = overlapping_rows(case)
    fam = {"empty": [], "all": list(range(P))}
    exact_after = set()
    if case[0] in ("planted", "decoys"):
        fam["shallow"] = [SUFFIX9, SUFFIX12, Q8_DUP]       # not p24, not Q x 11, the later copy of Q x 8
        fam["duplicate"] = [P16_DUP]                       # the later copy of the 16-byte pattern
        fam["long"] = [LONG]                               # the 600-byte pattern, longer than a window
        fam["odd"] = list(range(1, P, 2))
        # planted: pid 0 and the last pid (the long pattern), which ends a partial word; decoys: every pid at bit 31
        # and the last pid are decoys that never occur, so only bit 0 matches there (bit 31 matches in the dense case)
        fam["word_edges"] = word_edges(P)
        exact_after |= {"long", "word_edges"}             # nothing overlaps the long pattern or pid 0's occurrences
    elif case[0] == "dense":
        # matches are sparse here: the two sets also hold a pid whose every match a longer leftmost one hides
        _, data, offs = inputs(case)
        picked = Oracle(pats, "LeftmostLongest").scan_batch(data, offs)[2][:, 1]
        hidden = np.setdiff1d(rec[:, 1], picked).astype(np.int64)
        rng = np.random.default_rng(17)
        fam["one_percent"] = sorted(set(rng.choice(P, size=P // 100, replace=False).tolist()) | {int(hidden[0])})
        w = int(hidden[np.argmin(np.abs(hidden // 32 - (P // 32) // 2))]) // 32   # the word nearest the middle with one
        fam["middle_word"] = list(range(32 * w, min(32 * w + 32, P)))
        fam["word_edges"] = word_edges(P)
        fam["odd"] = list(range(1, P, 2))
    else:
        fam["core"] = [0]
        fam["children"] = list(range(1, P))                # the text's only matches end where a child's would
        fam["half_and_core"] = [0] + list(range(2, P, 2))
        exact_after.add("children")
    return tuple(fam), tuple(tuple(s) for s in fam.values()), frozenset(exact_after)


@functools.lru_cache(maxsize=None)
def assert_reach(case):
    """Each set reaches the corner it was built for (from the full overlapping rows), and for each set but empty, all
    and the listed exceptions some haystack's non-overlapping answer differs from the unfiltered one filtered to S."""
    pats, data, offs = inputs(case)
    names, sets, exact_after = family(case)
    rec = overlapping_rows(case).astype(np.int64)
    n, P = len(offs) - 1, len(pats)
    lens = np.array([len(p) for p in pats], dtype=np.int64)
    for name, S in zip(names, sets):
        adm = np.isin(rec[:, 1], np.asarray(S, dtype=np.int64))
        if name == "empty":
            continue
        assert adm.any(), name
        if name == "shallow":
            # some end has a longer pattern not admitted and a shorter admitted one: the walk passes the deepest node
            ends = {}
            for (h, p, s, e), a in zip(rec.tolist(), adm.tolist()):
                ends.setdefault((h, e), []).append((lens[p], a))
            assert any(any(not a1 and l1 > l2 for l1, a1 in v for l2, a2 in v if a2) for v in ends.values())
            # some occurrence has a lower pid (Q x 8, first copy) not admitted and a higher one admitted
            same = {}
            for (h, p, s, e), a in zip(rec.tolist(), adm.tolist()):
                same.setdefault((h, s, e), []).append((p, a))
            assert any(any(not a1 and p1 < p2 for p1, a1 in v for p2, a2 in v if a2) for v in same.values())
        if name == "duplicate":
            assert np.isin([P16, P16_DUP], rec[:, 1]).all()
        if name == "long":
            assert (rec[:, 1] == LONG).any()
        if name == "word_edges":
            assert ((rec[adm, 1] % 32) == 0).any()
            if case[0] == "dense":
                assert P % 32 == 0 and ((rec[adm, 1] % 32) == 31).any()
            if case[0] == "planted":
                assert P % 32 and (rec[:, 1] == P - 1).any()   # the last pid of a partial word
        if name == "all":
            continue
        wrong_after = False
        for kind in KINDS:
            _, _, full = Oracle(pats, kind.name).scan_batch(data, offs)
            post = full[np.isin(full[:, 1], np.asarray(S, dtype=np.uint32))]
            sub = subset_scan_batch(pats, kind, data, offs, sets, [names.index(name)] * n)[2]
            wrong_after |= not np.array_equal(post, sub)
        assert wrong_after == (name not in exact_after), name
    return True


@functools.lru_cache(maxsize=None)
def reference(case, kind_name, overlapping, r, codepoints):
    pats, data, offs = inputs(case)
    _, sets, _ = family(case)
    idx = (np.arange(len(offs) - 1) + r) % len(sets)
    return subset_scan_batch(pats, kind_name, data, offs, sets, idx, overlapping, codepoints)


def check_list(m, mo, total, want):
    wtotal, wcounts, wrec = want
    assert total == wtotal
    mo = mo.cpu().numpy()
    assert mo[0] == 0 and np.array_equal(np.diff(mo), wcounts.astype(np.int64))
    assert np.array_equal(m.cpu().numpy().view(np.uint32), wrec)


def check_filtered(case, want, codepoints=False, shift=0, r=0, idx64=False):
    """Every filtered query -- the lists of the three kinds and the overlapping search, find_first for every kind, both
    counts and is_match -- against subset_scan_batch with haystack h in set (h + r) % G, the geometry asserted after
    every call and list_records (the records stage 2 reserved) equal to the admitted overlapping total; then the "all"
    set against the unfiltered call, bit for bit."""
    assert assert_reach(case)
    pats, data, offs = inputs(case)
    names, sets, _ = family(case)
    G, n = len(sets), len(offs) - 1
    r %= G
    want = {**want, "pattern_sets": G}
    d, o = dev_at(data, shift), dev(offs)
    si = torch.from_numpy((np.arange(n) + r) % G).to(torch.int64 if idx64 else torch.int32).cuda()
    si_all = torch.full((n,), names.index("all"), dtype=si.dtype, device="cuda")
    admitted_over = reference(case, "Standard", True, r, False)[0]
    assert admitted_over > 0
    for kind in KINDS:
        ac = make_ac(pats, kind, codepoints)
        ps = ac.pattern_sets([list(s) for s in sets])
        kw = {"pattern_sets": ps, "set_index": si}
        for over in ((False, True) if kind == MatchKind.Standard else (False,)):
            ref = reference(case, kind.name, over, r, codepoints)
            check_list(*ac.scan_device(d, o, over, **kw), ref)
            assert_geometry(ac, want)
            assert ac._ac.last_stats["list_records"] == admitted_over, (kind, over)
            got = ac.count_matches_device(d, o, over, **kw).cpu().numpy()
            assert_geometry(ac, want)
            assert np.array_equal(got, ref[1].astype(np.int64)), (kind, over)
        ref = reference(case, kind.name, False, r, codepoints)
        got = ac.find_first_device(d, o, **kw).cpu().numpy()
        assert_geometry(ac, want)
        assert np.array_equal(got, first_rows_of(ref[1], ref[2])), kind
        if kind == MatchKind.Standard:
            got = ac.is_match_device(d, o, **kw).cpu().numpy()
            assert_geometry(ac, want)
            assert np.array_equal(got, reference(case, "Standard", True, r, False)[1] > 0)
        # the "all" set is the unfiltered call
        kw = {"pattern_sets": ps, "set_index": si_all}
        for over in ((False, True) if kind == MatchKind.Standard else (False,)):
            m0, mo0, t0 = ac.scan_device(d, o, over)
            m0, mo0 = m0.clone(), mo0.clone()
            m1, mo1, t1 = ac.scan_device(d, o, over, **kw)
            assert t0 == t1 and torch.equal(m0, m1) and torch.equal(mo0, mo1), (kind, over)
            assert torch.equal(ac.count_matches_device(d, o, over), ac.count_matches_device(d, o, over, **kw))
        assert torch.equal(ac.find_first_device(d, o), ac.find_first_device(d, o, **kw)), kind
        if kind == MatchKind.Standard:
            assert torch.equal(ac.is_match_device(d, o), ac.is_match_device(d, o, **kw))
            assert_geometry(ac, want)


# ---------------------------------------------------------------- W x R, planted batch
@pytest.mark.parametrize("ring", RINGS)
@pytest.mark.parametrize("w", range(1, 9))
def test_window_by_ring(monkeypatch, w, ring):
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_filtered(("planted", False), {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, shift=SHIFTS[(w + ring) % 3],
                       r=w + 3 * ring, idx64=bool((w + ring) % 2))


@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("w", (1, 4, 5, 8))
def test_window_by_ring_small_tasks(monkeypatch, w, ring):
    with geometry(monkeypatch, w, ring, 512):
        check_filtered(("planted", False), {"window": w, "ring": ring, "task_bytes": 512}, shift=SHIFTS[(w + ring) % 3],
                       r=w + ring, idx64=bool(w % 2))


@pytest.mark.parametrize("ring", RINGS)
@pytest.mark.parametrize("w", (1, 3, 4, 5, 8))
def test_code_points_window_by_ring(monkeypatch, w, ring):
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_filtered(("planted", True), {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, codepoints=True,
                       shift=SHIFTS[(w + ring) % 3], r=w + 2 * ring, idx64=bool((w + ring + 1) % 2))


# ---------------------------------------------------------------- filter budget
BUDGET_W = 5
BUDGETS = {
    "default": ("planted", None),
    "shallow": ("decoys", 8192),
    "saturated": ("dense", 4096),
}


@pytest.mark.parametrize("utf8", [False, True], ids=["bytes", "utf8"])
@pytest.mark.parametrize("task_bytes", (DEFAULT_TASK, 512))
@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("budget", list(BUDGETS))
def test_filter_budget(monkeypatch, budget, ring, task_bytes, utf8):
    name, nbytes = BUDGETS[budget]
    case = (name, utf8)
    smem = matcher._Automaton._smem_optin(torch.cuda.current_device())
    host_budget = nbytes if nbytes is not None else max(4096, smem - matcher._Automaton.SIEVE_SMEM_RESERVE)
    W, last_level, probes, bloom_bytes, fill = host_geometry(case, host_budget, BUDGET_W)
    assert W == BUDGET_W
    if budget == "default":
        assert last_level == 16
    elif budget == "shallow":
        assert last_level == W and fill < 0.05
    else:
        assert last_level == W and bloom_bytes == 4096 and fill >= 0.95, fill
    want = {"window": W, "last_level": last_level, "probes": probes, "bloom_bytes": bloom_bytes, "ring": ring,
            "task_bytes": task_bytes}
    with geometry(monkeypatch, BUDGET_W, ring, task_bytes, nbytes):
        check_filtered(case, want, codepoints=utf8, shift=SHIFTS[(ring + task_bytes // 512) % 3], r=ring + task_bytes // 512 + utf8,
                       idx64=bool((ring + utf8) % 2))


# ---------------------------------------------------------------- reverse-trie fan-out
@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("w", (1, 5, 8))
@pytest.mark.parametrize("fan", list(FANOUTS) + [TWO_LEVEL])
def test_trie_fanout(monkeypatch, fan, w, ring):
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_filtered(("fanout", fan), {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, shift=SHIFTS[w % 3], r=w + ring,
                       idx64=bool(w % 2))


# ---------------------------------------------------------------- capacity retry
@pytest.mark.parametrize("case", [("dense", False), ("planted", True)], ids=["dense", "planted-utf8"])
def test_capacity_retry(case):
    """capacity=1 on a fresh automaton: the first attempt has room for 1 024 records (the workspace's least), fewer
    than stage 2 reserves, so the list is scanned again with room for all of it.  Most haystacks search the "odd" set
    (every fourth one another set), which keeps more than 1 024 admitted overlapping records -- and, in the dense case,
    more than 1 024 rows of every non-overlapping kind.  Rows, total and the reservation (admitted pids only) are right
    after the retry, and the workspace grew to hold it."""
    assert assert_reach(case)
    pats, data, offs = inputs(case)
    names, sets, _ = family(case)
    n = len(offs) - 1
    idx = np.array([names.index("odd") if h % 4 != 3 else (h // 4) % len(sets) for h in range(n)])
    si = torch.from_numpy(idx).cuda()
    d, o = dev(data), dev(offs)
    admitted_over = subset_scan_batch(pats, "Standard", data, offs, sets, idx, True)[0]
    assert admitted_over > 1024
    with forced("sieve"):
        for kind in KINDS:
            for over in ((False, True) if kind == MatchKind.Standard else (False,)):
                want = subset_scan_batch(pats, kind, data, offs, sets, idx, over, case[1])
                if case[0] == "dense":
                    assert want[0] > 1024
                ac = make_ac(pats, kind, case[1])   # a fresh workspace for every call
                ps = ac.pattern_sets([list(s) for s in sets])
                check_list(*ac.scan_device(d, o, over, capacity=1, pattern_sets=ps, set_index=si), want)
                assert ac._ac.last_stats["list_records"] == admitted_over
                ws = ac._ac._ws[(torch.cuda.current_device(), 0)]
                assert ws["capacity"] >= max(want[0], admitted_over) > 1024   # the first attempt came back incomplete


# ---------------------------------------------------------------- early exits with sets
U = b"azb"   # a pattern no set of these tests admits, planted early in every haystack


def _skip_batch():
    rng = np.random.default_rng(9)
    n, L = 9, 1 << 20
    data = rng.integers(97, 101, size=n * L, dtype=np.uint8).astype(np.uint8)   # a..d: no pattern occurs by chance
    offs = np.arange(n + 1, dtype=np.int64) * L
    for h in range(n):
        data[h * L + 40:h * L + 43] = np.frombuffer(U, dtype=np.uint8)
    return data, offs


@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("shift", [0, 188, 511])
def test_preflagged_haystacks_are_skipped_exactly(variant, shift):
    """Unadmitted matches early in every haystack: they set no flag, so the pre-flags are all the kernel sees, and the
    skip counters are what the task grid predicts for them."""
    data, offs = _skip_batch()
    n, L = len(offs) - 1, 1 << 20
    pats = [b"abcz", b"zz", b"dcbaz", U]
    ac = BytesAhoCorasick(pats)
    ps = ac.pattern_sets([[0, 1, 2], [3]])
    si = torch.zeros(n, dtype=torch.int64 if shift % 2 else torch.int32, device="cuda")
    with forced(variant):
        d, o = dev_at(data, shift), dev(offs)
        pre = np.arange(n) % 2 == 0
        out = torch.from_numpy(pre.copy()).cuda()
        ac.is_match_device(d, o, out=out, pattern_sets=ps, set_index=si)
        assert out.cpu().numpy().tolist() == pre.tolist()
        st = ac._ac.last_stats
        T = st["task_bytes"]
        assert T == (512 if variant == "sieve-small-tasks" else 16384) and st["pattern_sets"] == 2
        tasks, windows = predicted_any_skips(d.data_ptr(), offs, pre, T)
        assert (st["tasks_skipped"], st["windows_skipped"]) == (tasks, windows)
        assert tasks > 0 and st["tasks"] == (n * L + (d.data_ptr() & 511) + T - 1) // T
        if shift and T > 512:
            assert windows > 0
        # nothing admitted occurs: nothing found, nothing skipped; the other set finds U everywhere
        fresh = ac.is_match_device(d, o, pattern_sets=ps, set_index=si)
        assert not fresh.any() and ac._ac.last_stats["tasks_skipped"] == ac._ac.last_stats["windows_skipped"] == 0
        assert ac.is_match_device(d, o, pattern_sets=ps, set_index=torch.ones_like(si)).all()
        # admitted matches where the unfiltered test plants them
        data2 = data.copy()
        data2[2 * L + 1000:2 * L + 1004] = np.frombuffer(b"abcz", dtype=np.uint8)
        data2[3 * L + 5:3 * L + 7] = np.frombuffer(b"zz", dtype=np.uint8)
        out = torch.from_numpy(pre.copy()).cuda()
        ac.is_match_device(dev_at(data2, shift), o, out=out, pattern_sets=ps, set_index=si)
        want = pre.copy()
        want[3] = True
        assert out.cpu().numpy().tolist() == want.tolist()


@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("kind", KINDS, ids=[k.name for k in KINDS])
@pytest.mark.parametrize("shift", [0, 188, 511])
def test_entry_keys_skip_exactly(variant, kind, shift):
    """Keys come only from admitted matches: the first call's keys are the subset's, and a second call with them as
    entry keys returns them unchanged and skips exactly what the task grid predicts from the subset's keys."""
    data, offs = _skip_batch()
    n, L = len(offs) - 1, 1 << 20
    pats = [b"abcz", b"zz", b"dcbaz", b"bcz", U]
    for h, at in ((0, 100), (2, 300_000), (3, 17_000), (4, L - 10), (6, 600_000), (7, 5)):
        data[h * L + at:h * L + at + 4] = np.frombuffer(b"abcz", dtype=np.uint8)
    data[6 * L + 800_000:6 * L + 800_002] = np.frombuffer(b"zz", dtype=np.uint8)
    sets = [[0, 1, 2, 3], [1, 3]]
    idx = np.arange(n) % 2
    ac = BytesAhoCorasick(pats, kind)
    ps = ac.pattern_sets(sets)
    flt = (ps, torch.from_numpy(idx).to(torch.int64 if shift % 2 else torch.int32).cuda())
    _, counts, rec = subset_scan_batch(pats, kind, data, offs, sets, idx)
    want = first_rows_of(counts, rec)
    assert (want[:, 0] >= 0).sum() >= 4 and (want[:, 0] < 0).any()
    with forced(variant):
        d, o = dev_at(data, shift), dev(offs)
        keys = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        ac._ac.first_keys(d, o, keys, flt)
        assert np.array_equal(ac._ac.first_rows(d, o, keys, flt).cpu().numpy(), want)
        key_hi = keys.cpu().numpy().view(np.uint64) >> np.uint64(32)
        want_hi = np.where(want[:, 0] >= 0, want[:, 2] if kind == MatchKind.Standard else want[:, 1], 0xFFFFFFFF)
        assert np.array_equal(key_hi.astype(np.int64), want_hi)
        again = keys.clone()
        scratch = ac._ac.first_keys(d, o, again, flt).cpu().tolist()
        assert torch.equal(again, keys)
        T = ac._ac._plan(d, n).task_bytes
        assert T == (512 if variant == "sieve-small-tasks" else 16384)
        tasks, windows = predicted_first_skips(d.data_ptr(), offs, want_hi, T, kind, ac._ac.max_pattern_len)
        assert (scratch[1], scratch[2]) == (tasks, windows)
        assert tasks > 0


@pytest.mark.parametrize("kind", KINDS, ids=[k.name for k in KINDS])
def test_one_large_haystack_stops_early(kind):
    """256 MiB, far more tasks than the grid has warps.  An unadmitted match at 700 and an admitted one at the end: the
    answer is the end.  With a set that admits the early match, more than half the tasks are skipped."""
    n = 256 << 20
    ac = BytesAhoCorasick([b"needle", b"haystack", b"needle in"], kind)
    ps = ac.pattern_sets([[1], [0, 1, 2]])
    late, early = (torch.tensor([g], dtype=dt, device="cuda") for g, dt in ((0, torch.int32), (1, torch.int64)))
    offs = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    hay = torch.full((n,), ord("x"), dtype=torch.uint8, device="cuda")
    put = lambda at, b: hay[at:at + len(b)].copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda())  # noqa: E731
    put(700, b"needle in")
    put(n - 8, b"haystack")
    with forced("sieve"):
        assert ac.find_first_device(hay, offs, pattern_sets=ps, set_index=late).cpu().tolist() == [[1, n - 8, n]]
        assert ac.is_match_device(hay, offs, pattern_sets=ps, set_index=late).cpu().tolist() == [True]
        want = {MatchKind.Standard: [0, 700, 706], MatchKind.LeftmostFirst: [0, 700, 706], MatchKind.LeftmostLongest: [2, 700, 709]}[kind]
        assert ac.find_first_device(hay, offs, pattern_sets=ps, set_index=early).cpu().tolist() == [want]
        st = ac._ac.last_stats
        assert st["skip_counters"].cpu().tolist()[1] > st["tasks"] // 2, st
        assert ac.is_match_device(hay, offs, pattern_sets=ps, set_index=early).cpu().tolist() == [True]
        st = ac._ac.last_stats
        assert st["tasks_skipped"] > st["tasks"] // 2, st
    del hay


# ---------------------------------------------------------------- set indices outside [0, n_sets)
INT32_MIN = -(1 << 31)
BAD_INDEX = {torch.int32: [-1, INT32_MIN, "G"], torch.int64: [-1, "G", 1 << 32, (1 << 32) + 1, (1 << 63) - 1]}


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["int32", "int64"])
@pytest.mark.parametrize("kind", KINDS, ids=[k.name for k in KINDS])
def test_indices_outside_the_sets_admit_nothing(kind, dtype):
    """Through the internal paths, which take (PatternSets, index) without the argument check.  The bitset has an
    all-patterns guard row on each side of the G real rows, and real set 0 matches everywhere: a lost bounds check, or
    an index cut to 32 bits (2^32 -> 0, 2^32 + 1 -> 1), reads a valid row and shows up as a wrong answer."""
    words = ["ab", "b", "abé", "é", "x"]
    pats = [w.encode() for w in words]
    P = len(pats)
    real = [list(range(P)), [1], [0, 3]]
    G = len(real)
    ac_b = make_ac(pats, kind)
    ac_s = make_ac(pats, kind, codepoints=True)
    bad = [G if v == "G" else v for v in BAD_INDEX[dtype]]
    idx = []
    for k, v in enumerate(bad):   # each bad index between two good ones
        idx += [k % G, v]
    idx.append(2)
    n = len(idx)
    hays = [("xxabé b " + "é" * (h % 3) + "ab").encode() for h in range(n)]
    data = np.frombuffer(b"".join(hays), dtype=np.uint8).copy()
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    d, o = dev(data), dev(offs)
    si = torch.tensor(idx, dtype=dtype, device="cuda")
    for ac in (ac_b, ac_s):
        ps = ac.pattern_sets([list(range(P))] + real + [list(range(P))])
        narrowed = PatternSets.__new__(PatternSets)
        narrowed.__dict__.update(ps.__dict__)
        narrowed.bits, narrowed.n_sets = ps.bits[1:1 + G], G
        assert narrowed.bits.data_ptr() == ps.bits.data_ptr() + 4 * ps.words
        flt = (narrowed, si)
        cp = ac is ac_s
        outside = np.array([not 0 <= v < G for v in idx])
        with forced("sieve"):
            for over in ((False, True) if kind == MatchKind.Standard else (False,)):
                ref = subset_scan_batch(pats, kind, data, offs, real, idx, over, cp)
                assert (ref[1][~outside] > 0).all() and not ref[1][outside].any()
                check_list(*ac._ac.scan_device(d, o, over, cp, flt=flt), ref)
                got = ac._ac.count_device(d, o, over, flt=flt).cpu().numpy()
                assert np.array_equal(got, ref[1].astype(np.int64)), over
            ref = subset_scan_batch(pats, kind, data, offs, real, idx)
            keys = torch.full((n,), -1, dtype=torch.int64, device="cuda")
            ac._ac.first_keys(d, o, keys, flt)
            assert (keys.cpu().numpy()[outside] == -1).all()
            assert np.array_equal(ac._ac.first_rows(d, o, keys, flt).cpu().numpy(), first_rows_of(ref[1], ref[2]))
            got = ac._ac.any_device(d, o, flt=flt).cpu().numpy()
            assert np.array_equal(got, ~outside)


# ---------------------------------------------------------------- streams at the seams
CUTS = (1, 7, 511, 512, 513, 16383, 16385)


def _chunks(hay: bytes, h, admitted, utf8):
    """hay cut at the sizes of CUTS (rotated by h) and inside each admitted occurrence (at character starts)."""
    cuts, at, k = set(), 0, h
    while at < len(hay):
        at += CUTS[k % len(CUTS)]
        k += 1
        cuts.add(min(at, len(hay)))
    cuts |= {(s + e) // 2 for s, e in admitted}
    cuts |= {s + 1 for s, e in admitted}
    if utf8:
        cuts = {c for c in cuts if c >= len(hay) or hay[c] & 0xC0 != 0x80}
    cuts = sorted(c for c in cuts if 0 < c < len(hay))
    return [hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])]


@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("utf8", [False, True], ids=["bytes", "utf8"])
@pytest.mark.parametrize("kind", KINDS, ids=[k.name for k in KINDS])
def test_streams_with_sets(kind, utf8, variant):
    case = ("planted", utf8)
    assert assert_reach(case)
    pats, data, offs = inputs(case)
    names, sets, _ = family(case)
    n, G = len(offs) - 1, len(sets)
    r = 1 + utf8 + 2 * KINDS.index(kind)
    idx = (np.arange(n) + r) % G
    hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(n)]
    over = subset_scan_batch(pats, "Standard", data, offs, sets, idx, True)[2]
    chunks = [_chunks(hays[h], h, [(int(s), int(e)) for _, _, s, e in over[over[:, 0] == h][:8].tolist()], utf8) for h in range(n)]
    assert all(b"".join(c) == hays[h] for h, c in enumerate(chunks))
    _, counts, rec = subset_scan_batch(pats, kind, data, offs, sets, idx, False, utf8)
    want_first = first_rows_of(counts, rec)
    ac = make_ac(pats, kind, utf8)
    ps = ac.pattern_sets([list(s) for s in sets])
    si = torch.from_numpy(idx).to(torch.int64 if utf8 else torch.int32).cuda()
    with forced(variant):
        im = ac.is_match_stream_batch(n, pattern_sets=ps, set_index=si)
        ff = ac.find_first_stream_batch(n, pattern_sets=ps, set_index=si)
        steps = max(len(c) for c in chunks)
        for t in range(steps):
            part = [c[t] if t < len(c) else b"" for c in chunks]
            po = np.zeros(n + 1, dtype=np.int64)
            np.cumsum([len(p) for p in part], out=po[1:])
            pd = torch.from_numpy(np.frombuffer(b"".join(part) + b"\0", dtype=np.uint8)[:po[-1]].copy()).cuda()
            last = torch.full((n,), t == steps - 1, dtype=torch.bool, device="cuda")
            flags = im.feed_device(pd, dev(po), last)
            rows = ff.feed_device(pd, dev(po), last)
        assert np.array_equal(flags.cpu().numpy(), counts > 0)
        assert np.array_equal(rows.cpu().numpy(), want_first)
        assert ac._ac.last_stats["pattern_sets"] == G


# ---------------------------------------------------------------- tokens
def _enc(seq):
    return b"".join(bytes([0x80 | (x >> 14), (x >> 7) & 0x7F, x & 0x7F]) for x in seq)


@pytest.mark.parametrize("dtype", [torch.uint16, torch.int32, torch.int64, "misaligned"])
@pytest.mark.parametrize("kind", KINDS, ids=[k.name for k in KINDS])
def test_token_queries_with_sets(kind, dtype):
    """TokenAhoCorasick's device queries with pattern_sets=, against the subset reference on the encoded bytes with
    positions divided by 3."""
    rng = np.random.default_rng(23 + KINDS.index(kind))
    vocab = np.array([5, 255, 256, 1000, 40000, 65535, 7, 9])
    pats = [rng.choice(vocab, size=int(rng.integers(1, 5))).tolist() for _ in range(40)]
    pats += [pats[3], pats[3], [7, 9, 5], [9, 5], [5]]   # duplicates, a nested family
    P = len(pats)
    sets = [[], list(range(P)), word_edges(P), [p for p in range(P) if rng.random() < 0.3], [P - 2, P - 1, 3]]
    hays = [rng.choice(vocab, size=int(rng.choice([0, 1, 5, 60, 700]))).tolist() for _ in range(37)]
    n = len(hays)
    idx = np.arange(n) % len(sets)
    lens = [len(h) for h in hays]
    toffs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=toffs[1:])
    flat = np.array([x for h in hays for x in h], dtype=np.int64)
    if dtype == "misaligned":
        buf = torch.zeros(len(flat) + 1, dtype=torch.int32, device="cuda")
        buf[1:] = torch.from_numpy(flat).cuda()
        toks = buf[1:]
    else:
        toks = torch.from_numpy(flat).to(dtype).cuda()
    o = dev(toffs)
    epats = [_enc(p) for p in pats]
    edata = np.frombuffer(b"".join(_enc(h) for h in hays) + b"\0", dtype=np.uint8)[:3 * len(flat)].copy()
    eoffs = toffs * 3
    ac = TokenAhoCorasick(pats, matchkind=kind)
    ps = ac.pattern_sets(sets)
    si = torch.from_numpy(idx).cuda()
    for over in ((False, True) if kind == MatchKind.Standard else (False,)):
        total, counts, rec = subset_scan_batch(epats, kind, edata, eoffs, sets, idx, over)
        rec = rec.astype(np.int64)
        rec[:, 2:] //= 3
        m, mo, t = ac.scan_device(toks, o, over, pattern_sets=ps, set_index=si)
        assert t == total and np.array_equal(np.diff(mo.cpu().numpy()), counts.astype(np.int64))
        assert np.array_equal(m.cpu().numpy().astype(np.int64), rec)
        got = ac.count_matches_device(toks, o, over, pattern_sets=ps, set_index=si).cpu().numpy()
        assert np.array_equal(got, counts.astype(np.int64))
        if over:
            assert np.array_equal(ac.is_match_device(toks, o, pattern_sets=ps, set_index=si).cpu().numpy(), counts > 0)
        else:
            assert total > 0
            assert np.array_equal(ac.find_first_device(toks, o, pattern_sets=ps, set_index=si).cpu().numpy(), first_rows_of(counts, rec))
