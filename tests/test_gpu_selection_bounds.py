"""GPU tests of the grid-wide selection at its pointer-jumping bounds (-m gpu).  A haystack whose overlapping list has
more than ACB_LONG_STRETCH records is selected by the whole grid: every record gets its successor NEXT(end), then
ceil_log2(longest stretch of the batch) rounds of pointer jumping count the chain (count_matches) or mark it
(count_matches_by_pattern, matching_patterns); acb_count_rows does the same over one haystack's int64 rows.  Both are
exact only if 2^rounds reaches the chain's length, which is tightest when every record of the longest stretch is
selected and its length is a power of two.

The inputs choose the chain length exactly: [a] over a * m (every record selected by every kind: chain = stretch = m),
[a, aa] over a * m (Standard and LeftmostFirst: chain m in a stretch of 2 m - 1; LeftmostLongest: ceil(m / 2)) for m
around 2^12, 2^13 and 2^14, each the longest stretch of its batch, next to short and empty haystacks, and nested,
self-overlapping patterns over a text whose chain is exactly 2^13 records.  Every query that selects on the grid runs at
16 KiB and 512-byte tasks, rings 1 and 8 and three offsets of the data from the task grid, against the oracle, with
last_stats' long_stretches asserted (an input that no longer reaches the grid fails instead of passing silently).  The
two row entry points get translated oracle lists that straddle 2^32, against the oracle and the Python chain model."""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, _capi, matcher  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, dev, dev_at  # noqa: E402
from .sieve_geometry_helpers import assert_geometry, geometry, hist_of, hits_of, hits_sums  # noqa: E402
from .stream_model import next_selected  # noqa: E402
from .test_count_cpu import count_by_chain  # noqa: E402
from .test_gpu_count import KIND_IDS, batch  # noqa: E402

L_STRETCH = _capi.ACB_LONG_STRETCH
CHAIN_MS = (4096, 4097, 8191, 8192, 8193, 16384)   # 4096: [a]'s last stretch on the one-thread path
NESTED = [b"ab", b"aba", b"bab", b"abab", b"b", b"baab", b"aa", b"ab"]
NESTED_CHAIN = 1 << 13
SETS = {"a": [b"a"], "a_aa": [b"a", b"aa"], "nested": NESTED}
SHIFTS = (0, 1, 511)


def shorts(rng, k):
    """k short haystacks over a, b, x (some empty) and one empty haystack."""
    return [bytes(rng.choice(list(b"abx"), size=int(rng.integers(0, 40))).astype(np.uint8)) for _ in range(k)] + [b""]


@functools.lru_cache(maxsize=None)
def nested_haystack(kind):
    """A text over a, b whose selection under NESTED and `kind` is exactly NESTED_CHAIN records: the shortest prefix of
    a seeded text that the oracle gives that many, confirmed by the successor chain's pointer jumping (count_by_chain)."""
    text = np.random.default_rng(71).choice(list(b"ab"), size=8 * NESTED_CHAIN).astype(np.uint8).tobytes()
    orc = Oracle(NESTED, kind.value)
    lo, hi = 0, len(text)
    while lo < hi:
        mid = (lo + hi) // 2
        if len(orc.find(text[:mid])) < NESTED_CHAIN:
            lo = mid + 1
        else:
            hi = mid
    hay = text[:lo]
    assert len(orc.find(hay)) == NESTED_CHAIN
    over = Oracle(NESTED, 0).find(hay, overlapping=True)
    assert count_by_chain(kind.value, over, max(map(len, NESTED))) == NESTED_CHAIN and len(over) > 2 * L_STRETCH
    return hay


@functools.lru_cache(maxsize=None)
def batches(name, kind):
    """-> [(data, offs, expected chain per chain haystack)]: for [a] and [a, aa] one batch per m of CHAIN_MS, holding a * m'
    for every m' <= m (so a * m is the batch's longest stretch; the last batch holds all of them) between short and
    empty haystacks; for NESTED one batch around the kind's nested haystack."""
    rng = np.random.default_rng(17)
    if name == "nested":
        return [batch(shorts(rng, 20) + [nested_haystack(kind)] + [b"babab" * 10] + shorts(rng, 20))]
    out = []
    for k in range(len(CHAIN_MS)):
        hays = []
        for m in CHAIN_MS[:k + 1]:
            hays += shorts(rng, 10) + [b"a" * m]
        out.append(batch(hays + shorts(rng, 10)))
    return out


@functools.lru_cache(maxsize=None)
def automaton(name, kind):
    return BytesAhoCorasick(SETS[name], kind)


@functools.lru_cache(maxsize=None)
def expected(name, kind, b, overlapping):
    data, offs = batches(name, kind)[b]
    pats = SETS[name]
    _, counts, rec = Oracle(pats, kind.value).scan_batch(data, offs, overlapping=overlapping)
    _, over_counts, _ = Oracle(pats, 0).scan_batch(data, offs, overlapping=True, want_records=False)
    return counts.astype(np.int64), rec, int((over_counts > L_STRETCH).sum()), int(over_counts.sum())


def test_inputs_reach_their_chain_lengths():
    """The construction the grid tests rely on, on the host: chain lengths and which haystacks go to the grid."""
    for kind in KINDS:
        for name in ("a", "a_aa"):
            counts, _, n_long, _ = expected(name, kind, len(CHAIN_MS) - 1, False)
            chains = counts[np.diff(batches(name, kind)[-1][1]) >= CHAIN_MS[0]]   # every a * m, in order
            halve = name == "a_aa" and kind == MatchKind.LeftmostLongest
            assert chains.tolist() == [(m + 1) // 2 if halve else m for m in CHAIN_MS]
            assert n_long == (len(CHAIN_MS) - 1 if name == "a" else len(CHAIN_MS))   # [a]'s 4096 records stay off the grid
        counts, _, n_long, _ = expected("nested", kind, 0, False)
        assert n_long == 1 and NESTED_CHAIN in counts.tolist()


@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("ring", (1, 8))
@pytest.mark.parametrize("task_bytes", (16384, 512))
@pytest.mark.parametrize("name", list(SETS))
def test_grid_selection_at_its_bounds(monkeypatch, name, task_bytes, ring, shift):
    """count_matches, count_matches_by_pattern, matching_patterns and the match list of every kind (and the
    overlapping hits and list of Standard) on each batch, against the oracle."""
    want = {"ring": ring, "task_bytes": task_bytes}
    with geometry(monkeypatch, matcher._Automaton.SIEVE_W_MAX, ring, task_bytes):
        for kind in KINDS:
            ac = automaton(name, kind)
            pats = SETS[name]
            for b, (data, offs) in enumerate(batches(name, kind)):
                d, o = dev_at(data, shift), dev(offs)
                n = len(offs) - 1
                for overlapping in ([False, True] if kind == MatchKind.Standard else [False]):
                    counts, rec, n_long, over_total = expected(name, kind, b, overlapping)
                    where = (name, kind, b, overlapping)
                    grid = n_long if not overlapping else 0   # the overlapping counts run the sieve kernel, no epilogue
                    got = ac.count_matches_device(d, o, overlapping).cpu().numpy()
                    st = ac._ac.last_stats
                    assert_geometry(ac, want)
                    assert st["mode"] == "count" and st["long_stretches"] == grid, (where, st)
                    assert np.array_equal(got, counts), where
                    hist = ac.count_matches_by_pattern_device(d, o, overlapping).cpu().numpy()
                    st = ac._ac.last_stats
                    assert_geometry(ac, want)
                    assert st["mode"] == "pattern_counts" and st["long_stretches"] == grid, (where, st)
                    assert np.array_equal(hist, hist_of(rec, len(pats))), where
                    hits = [t.cpu().numpy() for t in ac.matching_patterns_device(d, o, overlapping)]
                    st = ac._ac.last_stats
                    assert_geometry(ac, want)
                    assert st["mode"] == "matching_patterns" and st["long_stretches"] == n_long and st["rows"] == n_long, (where, st)
                    for t, exp in zip(hits, hits_of(rec, n, len(pats))):
                        assert np.array_equal(t, exp), where
                    rows, cols = hits_sums(hits, n, len(pats))
                    assert np.array_equal(rows, got) and np.array_equal(cols, hist), where
                    m, mo, total = ac.scan_device(d, o, overlapping)
                    assert_geometry(ac, want)
                    assert ac._ac.last_stats["list_records"] == over_total, where
                    assert total == len(rec) and np.array_equal(np.diff(mo.cpu().numpy()), counts), where
                    assert np.array_equal(m.cpu().numpy().view(np.uint32), rec), where


# ---------------------------------------------------------------- acb_select_non_overlapping and acb_count_rows
TRANSLATE = (1 << 32) - 7   # every position moves by this much: the rows straddle 2^32, the selection does not change


def row_cases():
    """(patterns, haystack) pairs: [a] chains of 0, 1, 2, 2^k - 1, 2^k and 2^k + 1 records for k up to 14, [a, aa]
    at the same bounds, and seeded mixed sets with duplicates, nested and self-overlapping patterns."""
    ns = sorted({0, 1, 2} | {(1 << k) + d for k in range(2, 15) for d in (-1, 0, 1)})
    cases = [([b"a"], b"a" * n) for n in ns]
    cases += [([b"a", b"aa"], b"a" * n) for n in ns if n >= 1 << 12]
    rng = np.random.default_rng(404)
    for c in range(40):
        alpha = b"abc" if c % 3 else b"ab"
        pats = [bytes(rng.choice(list(alpha), size=int(rng.integers(1, 6))).astype(np.uint8)) for _ in range(int(rng.integers(2, 9)))]
        pats += [pats[int(rng.integers(0, len(pats)))], pats[0] + pats[-1], b"a" * int(rng.integers(1, 4))]
        cases.append((pats, bytes(rng.choice(list(alpha), size=int(rng.integers(1, 3000))).astype(np.uint8))))
    return cases


def chain_rows(over, kind, max_len):
    """The selection as the Python chain model follows it: NEXT(0), NEXT(end of that), ... (stream_model.next_selected)."""
    ends = [e for _, _, e in over]
    picked, j = [], next_selected(over, ends, 0, max_len, kind)
    while j is not None:
        picked.append(over[j])
        j = next_selected(over, ends, over[j][2], max_len, kind)
    return picked


def as_rows(recs):
    rows = np.zeros((len(recs), 4), dtype=np.int64)
    if recs:
        rows[:, 1:] = np.asarray(recs, dtype=np.int64)
        rows[:, 2:] += TRANSLATE
    return rows


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_row_selection_and_count_across_2_32(kind):
    for pats, hay in row_cases():
        ac = BytesAhoCorasick(pats, kind)
        a = ac._ac
        max_len = max(map(len, pats))
        over = Oracle(pats, 0).find(hay, overlapping=True)
        assert over == sorted(over, key=lambda r: (r[2], r[1], r[0]))   # the rows' order: end, start, pattern
        want = Oracle(pats, kind.value).find(hay)
        shifted = [(p, s + TRANSLATE, e + TRANSLATE) for p, s, e in over]
        assert chain_rows(shifted, kind.value, max_len) == [(p, s + TRANSLATE, e + TRANSLATE) for p, s, e in want]
        assert count_by_chain(kind.value, shifted, max_len) == len(want)
        n = len(over)
        rows = dev(as_rows(over))
        out = torch.full((max(n, 1), 4), -1, dtype=torch.int64, device="cuda")
        count = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        assert a._L.acb_select_non_overlapping(a._h, rows.data_ptr() if n else None, n, out.data_ptr(), count.data_ptr(),
                                               stream) == _capi.ACB_OK, _capi.last_error()
        k = int(count.item())
        assert k == len(want), (pats, len(hay))
        assert np.array_equal(out[:k].cpu().numpy(), as_rows(want)), (pats, len(hay))
        scratch = torch.empty((max(n, 1), 2), dtype=torch.int64, device="cuda")   # 16 bytes per row
        rc = a._L.acb_count_rows(a._h, rows.data_ptr() if n else None, n, scratch.data_ptr(), count.data_ptr(), stream)
        assert rc == _capi.ACB_OK, _capi.last_error()
        assert int(count.item()) == k, (pats, len(hay))
