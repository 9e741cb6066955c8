"""GPU edge-case tests (-m gpu): inputs built to reach the paths of the scan kernels and their epilogues that
ordinary text reaches rarely or never -- code points spread over many segments, matches running past segment
ends, the repair pass, haystack and match boundaries on the segment and task grid, patterns longer than the filter
window, a segment or a task, the full byte range, the two ways of computing per-haystack offsets, a result that does
not fit the first buffer, and one workspace reused across different scans.  Every kernel variant, compared with the
CPU oracle bit for bit.  Where a test is aimed at one path it also checks, from the scan's statistics, that the
input got there: a changed default (segment size, span of the near code-point fix-up, records per haystack of the
run-fill) must not quietly turn it into a test of something else."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind  # noqa: E402
from ahocorasick_rs_b200.matcher import PATH_FAR_CP, PATH_REPAIRED, PATH_SEARCH  # noqa: E402

from .gpu_helpers import (KINDS, SEARCH_IDS, SEARCHES, VARIANTS, check_batch, dev_at, forced, is_segmented,  # noqa: E402,F401
                          is_sieve, kernel, make_ac)

ALPHA = ["a", "b", "é", "—", "☃", "𝄞"]   # 1, 1, 2, 3, 3 and 4 bytes


def batch(hays):
    """list of bytes / str -> (uint8 data, int64 offsets)"""
    raw = [h.encode() if isinstance(h, str) else h for h in hays]
    offs = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=offs[1:])
    data = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)[: offs[-1]].copy()
    return data, offs


def text(rng, n, alphabet=ALPHA):
    return "".join(rng.choice(alphabet, size=n)) if n else ""


def planned_segment(variant, max_len):
    """The segment size acb_plan_scan picks: the tuning knob (1 KiB by default), at least 8 warm-ups, 64-aligned."""
    warm = max(16, (max_len + 15) & ~15)
    return (max(VARIANTS[variant][2] or 1024, 8 * warm) + 63) & ~63


def stats(ac, variant):
    st = ac._ac.last_stats
    assert st["engine"] == ("sieve" if is_sieve(variant) else "table")
    return st


def utf8_patterns(rng):
    """1 to 6 characters, beginning and ending with characters of every width, plus duplicates."""
    pats = set()
    for a in ALPHA:
        for b in ALPHA:
            pats.add(a + text(rng, int(rng.integers(0, 5))) + b)
    pats.update(text(rng, int(rng.integers(1, 4))) for _ in range(10))
    pats = sorted(pats)
    return [p.encode() for p in pats + pats[:4]]


# ---------------------------------------------------------------- a. ragged UTF-8 batches, code points
def ragged_utf8(variant, far, seed):
    """A batch whose haystacks all end within 4 segments of their start (the near fix-up), or one with haystacks
    longer than 12 segments (the far fix-up).  Lengths are in characters of 1 to 4 bytes."""
    rng = np.random.default_rng(seed)
    pats = utf8_patterns(rng)
    S = planned_segment(variant, max(len(p) for p in pats)) if not is_sieve(variant) else 1024
    lens = list(rng.integers(0, 3 * S // 4 + 1, size=120 if not far else 30))
    lens[::17] = [0] * len(lens[::17])
    if far:
        lens[3] = lens[11] = 12 * S
        lens[-1] = 13 * S + 7
    return pats, *batch([text(rng, int(n)) for n in lens])


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
def test_ragged_utf8_codepoints(kind, overlapping, far, kernel):
    pats, data, offs = ragged_utf8(kernel, far, seed=101 + far)
    ac = make_ac(pats, kind, codepoints=True)
    assert check_batch(pats, kind, data, offs, overlapping, codepoints=True, ac=ac) > 500
    st = stats(ac, kernel)
    if is_segmented(kernel):
        assert bool(st["paths"] & PATH_FAR_CP) == far


# ---------------------------------------------------------------- b. overrun, skipped head and repair, code points
def multibyte_runs(rng, n_runs):
    """Long runs of one multibyte character, rare ASCII separators."""
    parts = []
    for _ in range(n_runs):
        parts.append(rng.choice(["é", "☃", "𝄞"]) * int(rng.integers(20, 300)))
        parts.append(rng.choice(["x", " ", "é☃", ""]))
    return "".join(parts)


@pytest.mark.parametrize("kind", KINDS[1:], ids=lambda k: k.name)
def test_leftmost_runs_overrun_segments(kind, kernel):
    """Leftmost matches that are long runs of a multibyte character: matches run past segment ends across
    continuation bytes, warm-ups end inside a match (the head piece is skipped), speculated starts are wrong."""
    rng = np.random.default_rng(202)
    pats = [p.encode() for p in ["é" * 8, "é" * 3, "☃" * 5, "☃" * 2, "𝄞" * 4, "𝄞", "é☃", "x"]]   # at most 16 bytes
    hays = [multibyte_runs(rng, 400)] + [multibyte_runs(rng, int(rng.integers(1, 12))) for _ in range(60)]
    data, offs = batch(hays)
    ac = make_ac(pats, kind, codepoints=True)
    assert check_batch(pats, kind, data, offs, codepoints=True, ac=ac) > 5000
    st = stats(ac, kernel)
    if is_segmented(kernel):
        assert st["segment_bytes"] == planned_segment(kernel, 16)
        assert st["repairs"] > 0 and st["paths"] & PATH_REPAIRED


def test_dense_self_overlapping_codepoints(kernel):
    """'éé' on a run of 'é' after one to three ASCII characters: the code point counterpart of
    test_dense_self_overlapping_matches_single_haystack.  Guessed restart phases are wrong wherever the run's
    byte phase differs from the segment grid's."""
    pats = ["éé".encode()]
    repairs = 0
    for lead in (1, 2, 3):
        data, offs = batch(["b" * lead + "é" * 20_001, "é" * 777, "b" + "é" * 3001])
        ac = make_ac(pats, MatchKind.Standard, codepoints=True)
        assert check_batch(pats, MatchKind.Standard, data, offs, codepoints=True, ac=ac) > 10_000
        st = stats(ac, kernel)
        if is_segmented(kernel):
            repairs += st["repairs"]
            assert st["repairs"] == 0 or st["paths"] & PATH_REPAIRED
    if is_segmented(kernel):
        assert repairs > 0


# ---------------------------------------------------------------- c. boundaries on the segment and task grid
GRID_PATTERNS = {False: [b"q", b"ab", b"abcd", b"da", b"bcdefg"], True: [p.encode() for p in ["q", "é☃", "é☃𝄞é", "éé", "☃𝄞é"]]}
GRID_FILL = {False: ["x", "y", "a", "d"], True: ["x", "ñ", "é", "☃", "𝄞"]}


def fill(rng, nbytes, alphabet):
    out, left = [], nbytes
    while left:
        c = rng.choice([a for a in alphabet if len(a.encode()) <= left])
        out.append(c)
        left -= len(c.encode())
    return "".join(out).encode()


def grid_batch(S, mis, codepoints, rng):
    """Grid line k lies at byte k S - mis of the data.  Lines 1-3: haystack boundaries at line - 1, line, line + 1
    (with a pattern ending at it, one starting at it, and a pattern made of the bytes around it); lines 4-6: match
    starts; lines 7-9: match ends."""
    P = GRID_PATTERNS[codepoints][2]
    items, cuts = [], [0]
    for k in range(1, 10):
        pos = k * S - mis + (k - 1) % 3 - 1
        if k <= 3:
            items += [(pos - len(P), P), (pos, P)]
            cuts.append(pos)
        elif k <= 6:
            items.append((pos, P))
        else:
            items.append((pos - len(P), P))
    end = 10 * S - mis + 3
    raw, at = [], 0
    for pos, p in items:
        raw += [fill(rng, pos - at, GRID_FILL[codepoints]), p]
        at = pos + len(p)
    raw.append(fill(rng, end - at, GRID_FILL[codepoints]))
    data = np.frombuffer(b"".join(raw), dtype=np.uint8).copy()
    return data, np.array(cuts + [end], dtype=np.int64)


@pytest.mark.parametrize("codepoints", [False, True], ids=["bytes", "codepoints"])
def test_boundaries_on_the_grid(codepoints, kernel):
    rng = np.random.default_rng(303)
    pats = GRID_PATTERNS[codepoints]
    sieve = is_sieve(kernel)
    align = 511 if sieve else 63
    for shift in (0, 1, 63, 200):
        probe = dev_at(np.zeros(16, dtype=np.uint8), shift)
        mis = probe.data_ptr() & align
        assert mis == shift & align   # (fresh allocations are 512-byte aligned: the shift places the grid)
        for kind, overlapping in SEARCHES:
            ac = make_ac(pats, kind, codepoints)
            ac.scan_device(probe, torch.tensor([0, 16], dtype=torch.int64, device="cuda"))
            S = stats(ac, kernel)["task_bytes" if sieve else "segment_bytes"]
            if kernel == "sieve-small-tasks":
                assert S == 512
            data, offs = grid_batch(S, mis, codepoints, rng)
            assert check_batch(pats, kind, data, offs, overlapping, codepoints, ac=ac, shift=shift) >= 12
            assert stats(ac, kernel)["task_bytes" if sieve else "segment_bytes"] == S


# ---------------------------------------------------------------- d. long patterns
LONG = (16, 17, 64, 200, 511, 512, 513, 1500)


def long_pattern_batch(minlen, codepoints, seed):
    """Long patterns that are prefixes and suffixes of one base string (so they nest), mixed with short ones whose
    shortest is `minlen` bytes; text with full occurrences, near-misses sharing a long prefix or suffix, and nested
    occurrences, in a few haystacks."""
    rng = np.random.default_rng(seed)
    alpha = ["a", "b", "é", "☃", "𝄞"] if codepoints else ["a", "b", "c", "d"]
    base = text(rng, 1500, alpha).encode()

    def cut(b, n, tail=False):   # n bytes of b (whole characters only)
        if tail:
            i = len(b) - n
            while codepoints and i < len(b) and (b[i] & 0xC0) == 0x80:
                i += 1
            return b[i:]
        while codepoints and n < len(b) and (b[n] & 0xC0) == 0x80:
            n -= 1
        return b[:n]

    longs = [cut(base, n) for n in LONG] + [cut(base, n, tail=True) for n in (17, 200, 513)]
    shorts = [b"a" * minlen] + [text(rng, int(rng.integers(1, 4)), alpha).encode() for _ in range(30)]
    shorts = [s for s in shorts if len(s) >= minlen]
    pats = sorted(set(longs + shorts), key=lambda p: (len(p), p))
    pats = [pats[i] for i in rng.permutation(len(pats))]
    hays = []
    for _ in range(2):
        parts = []
        for p in longs:
            parts += [text(rng, int(rng.integers(0, 100)), alpha).encode(), p,                      # full
                      text(rng, int(rng.integers(0, 40)), alpha).encode(), cut(p, len(p) - 1) + b"Z",  # shares the prefix
                      b"Z" + cut(p, len(p) - 1, tail=True), b"x" + base + b"y"]                     # the suffix; nested
        hays.append(b"".join(parts))
    return pats, *batch(hays)


@pytest.mark.parametrize("codepoints", [False, True], ids=["bytes", "codepoints"])
@pytest.mark.parametrize("minlen", range(1, 10))
def test_long_patterns(minlen, codepoints, kernel):
    pats, data, offs = long_pattern_batch(minlen, codepoints, seed=400 + minlen)
    longest = max(len(p) for p in pats)
    assert min(len(p) for p in pats) == minlen and 1496 <= longest <= 1500
    for kind, overlapping in SEARCHES:
        ac = make_ac(pats, kind, codepoints)
        assert check_batch(pats, kind, data, offs, overlapping, codepoints, ac=ac) > 40
        st = stats(ac, kernel)
        if not is_sieve(kernel):
            assert st["segment_bytes"] >= 8 * ((longest + 15) & ~15) and st["segment_bytes"] == planned_segment(kernel, longest)


# ---------------------------------------------------------------- e. the full byte range
def random_bytes_batch(pats, seed, n=60, size=4000):
    rng = np.random.default_rng(seed)
    hays = []
    for _ in range(n):
        h = bytearray(rng.integers(0, 256, size=int(rng.integers(0, size)), dtype=np.uint8).tobytes())
        for _ in range(int(rng.integers(0, 12))):
            p = pats[int(rng.integers(0, len(pats)))]
            at = int(rng.integers(0, len(h) + 1))
            h[at:at] = p
        hays.append(bytes(h))
    return batch(hays)


ASCII_PATS = [b"the", b"a", b"zq", b"hello", b"lo w", b"~~", b"0123456789", b"\x7f"]
BINARY_PATS = [b"\x00", b"\x80", b"\xff\xff", b"\x00\x80\xff", b"\xc3\xa9", b"a\x00", b"\xfe\xff\x00\x01"]


@pytest.mark.parametrize("pats", [ASCII_PATS, BINARY_PATS], ids=["ascii-patterns", "binary-patterns"])
@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
def test_full_byte_range(pats, kind, overlapping, kernel):
    data, offs = random_bytes_batch(pats, seed=505 + len(pats))
    ac = make_ac(pats, kind)
    assert check_batch(pats, kind, data, offs, overlapping, ac=ac) > 300
    stats(ac, kernel)


from hypothesis import given, settings, strategies as st  # noqa: E402

PROPERTY_VARIANTS = ["staged-small-segments", "global-small-segments", "staged-byte-table-tiny", "staged-two-per-lane-tiny",
                     "sieve-small-tasks"]


@pytest.mark.parametrize("variant", PROPERTY_VARIANTS)
@settings(max_examples=30, deadline=None)
@given(st.binary(), st.binary(min_size=1), st.binary())
def test_bytes_extensive_forced(variant, prefix, pattern, suffix):
    """test_bytes_extensive_like_the_reference under forced kernel variants."""
    haystack = prefix + pattern + suffix
    with forced(variant):
        idx = BytesAhoCorasick([pattern]).find_matches_as_indexes(haystack)
    assert {i for (i, _, _) in idx} == {0}
    assert {haystack[s:e] for (_, s, e) in idx} == {pattern}
    assert idx[0][1] == haystack.find(pattern)


@pytest.mark.parametrize("variant", PROPERTY_VARIANTS)
@settings(max_examples=30, deadline=None)
@given(st.text(), st.text(min_size=1), st.text())
def test_unicode_extensive_forced(variant, prefix, pattern, suffix):
    """test_unicode_extensive_like_the_reference under forced kernel variants."""
    haystack = prefix + pattern + suffix
    with forced(variant):
        idx = AhoCorasick([pattern]).find_matches_as_indexes(haystack)
    assert {i for (i, _, _) in idx} == {0}
    assert {haystack[s:e] for (_, s, e) in idx} == {pattern}
    assert idx[0][1] == haystack.find(pattern)


# ---------------------------------------------------------------- f. per-haystack offsets
def counted(counts):
    """One haystack per entry: that many 'a's among 'b's; None = an empty haystack."""
    return batch([b"" if c is None else b"b" + b"ab" * c for c in counts])


def offsets_cases():
    rng = np.random.default_rng(606)
    nh = 50
    k = 4 * (nh + 1)   # the most records the run-fill takes
    few = list(np.bincount(rng.integers(0, nh, size=k), minlength=nh))
    more = list(few)
    more[int(rng.integers(0, nh))] += 1
    mid = list(rng.integers(0, 3, size=100))
    runs = [0] * 70 + mid[:50] + [None] * 70 + [0] * 70 + mid[50:] + [None] * 70 + [0] * 70
    return {
        "run-fill-limit": (few, False),
        "search-above-limit": (more, True),
        "matchless-runs": (runs, False),
        "empty-runs": ([None] * 80 + mid + [None] * 80, False),
        "first-only": ([300] + [0] * 200, False),
        "last-only": ([0] * 200 + [300], False),
        "first-only-many": ([5000] + [0] * 200, True),
        "last-only-many": ([None] * 200 + [5000], True),
        "none": (list(rng.choice([0, None], size=100_000)), False),
    }


OFFSETS_CASES = offsets_cases()


@pytest.mark.parametrize("case", list(OFFSETS_CASES))
def test_match_offsets(case, kernel):
    counts, search = OFFSETS_CASES[case]
    data, offs = counted(counts)
    pats = [b"a"]
    for overlapping in (False, True):
        ac = make_ac(pats, MatchKind.Standard)
        total = check_batch(pats, MatchKind.Standard, data, offs, overlapping, ac=ac)
        assert total == sum(c or 0 for c in counts)
        st = stats(ac, kernel)
        if not is_sieve(kernel):
            assert bool(st["paths"] & PATH_SEARCH) == search


# ---------------------------------------------------------------- g. a result larger than the first buffer
def capacity_inputs():
    rng = np.random.default_rng(707)
    far_pats, far_data, far_offs = ragged_utf8("staged", True, seed=708)
    return {
        # (patterns, data, offsets, code points, what a segment kernel must have done on a non-overlapping search)
        "bytes-repair": ([b"aa"], *batch([b"b" + b"a" * 20_001, b"a" * 5000]), False, PATH_REPAIRED),
        "codepoints-repair": (["éé".encode()], *batch(["bb" + "é" * 20_001, "é" * 5000]), True, PATH_REPAIRED),
        "codepoints-far": (far_pats, far_data, far_offs, True, PATH_FAR_CP),
        "bytes-ragged": ([b"a", b"ab", b"ba", b"bab", b"c"], *batch([text(rng, int(n), ["a", "b", "c"]).encode()
                                                                     for n in rng.integers(0, 800, size=200)]), False, 0),
    }


CAPACITY_INPUTS = capacity_inputs()


@pytest.mark.parametrize("name", list(CAPACITY_INPUTS))
@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
def test_capacity_one(name, kind, overlapping, kernel):
    pats, data, offs, codepoints, path = CAPACITY_INPUTS[name]
    ac = make_ac(pats, kind, codepoints)
    total = check_batch(pats, kind, data, offs, overlapping, codepoints, ac=ac, capacity=1)
    assert total > 1024
    ws = ac._ac._ws[(torch.cuda.current_device(), 0)]
    assert ws["capacity"] >= total > 1024   # the first attempt (room for 1 024 rows) came back incomplete
    st = stats(ac, kernel)
    if is_segmented(kernel) and not overlapping:
        assert st["paths"] & path == path


# ---------------------------------------------------------------- h. one workspace, many scans
@pytest.mark.parametrize("table,sieve", [("staged-small-segments", "sieve"), ("global-small-segments", "sieve-small-tasks"),
                                         ("staged-two-per-lane-tiny", "sieve"), ("staged", "sieve-small-tasks")])
def test_one_workspace_many_scans(table, sieve):
    """A fixed sequence of different scans through one automaton and one workspace slot, switching between a table
    walker and the sieve: every scan must leave the workspace's counters as the next one expects them."""
    rng = np.random.default_rng(808)
    pat_strs = ["éé", "a☃", "𝄞b", "ab", "b—é"]
    pats = [p.encode() for p in pat_strs]
    ac = AhoCorasick(pat_strs)
    S = planned_segment(table, max(len(p) for p in pats))
    alpha = ["a", "b", "é", "☃", "𝄞", "—"]
    far = batch([text(rng, int(n), alpha) for n in [12 * S, 40, 0, 13 * S, 500]])
    near = batch([text(rng, int(n), alpha) for n in rng.integers(0, S // 4, size=300)])
    repair = batch(["bb" + "é" * 20_001, "é" * 3000])
    # haystacks of exactly one segment each, on the grid (a fresh allocation is 512-byte aligned): nothing to repair
    clean = batch([fill(rng, S, alpha) for _ in range(40)])
    ws_key = (torch.cuda.current_device(), 0)

    def step(data_offs, variant, overlapping=False, capacity=None):
        with forced(variant):
            total = check_batch(pats, MatchKind.Standard, *data_offs, overlapping, codepoints=True, ac=ac, capacity=capacity)
        return total, stats(ac, variant)

    _, st = step(far, table)
    assert st["paths"] & PATH_FAR_CP
    _, st = step(near, table)
    assert not st["paths"] & PATH_FAR_CP
    _, st = step(repair, table)
    assert st["repairs"] > 0 and st["paths"] & PATH_REPAIRED
    _, st = step(clean, table)
    assert st["repairs"] == 0 and not st["paths"] & (PATH_REPAIRED | PATH_FAR_CP)
    # more matches than the workspace has room for, then a step that fits
    cap0 = ac._ac._ws[ws_key]["capacity"]
    big = batch(["ab" * (cap0 // 2 + 3000) + "é" * (cap0 + 5), "a☃" * 2000])
    total, _ = step(big, sieve)
    assert total > cap0 and ac._ac._ws[ws_key]["capacity"] > cap0
    cap1 = ac._ac._ws[ws_key]["capacity"]
    step(near, sieve)
    assert ac._ac._ws[ws_key]["capacity"] == cap1
    step(far, table, overlapping=True)
    step(far, table)
