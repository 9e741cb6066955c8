"""GPU tests of the host-buffer layer (-m gpu): host memory in, the scan, host lists out.  Every drop-in call goes
through one of three pieces of host code in matcher.py, each driving the kernels with its own buffers:
  * the lean one-haystack path (_small_call): a fixed workspace of 4096 rows for haystacks of up to SMALL_CALL_BYTES,
    the status words and the first SMALL_CALL_ROWS rows in one copy, and a hand-over to the general path when the
    list does not fit or the plan outgrows what was allocated;
  * scan_host's runs: the copy of run i+1 overlapping the scan of run i on two buffers and two workspace slots, a run
    whose list overflowed scanned again, haystack ids rebased to the batch;
  * the host batches (is_match, find_first, count_matches, count_matches_by_pattern, matching_patterns): offsets and
    bytes gathered into one grow-only pinned staging buffer and sent in one copy.
Every result is compared with the CPU oracle on the same bytes, small haystacks with the brute-force statement
(tests/spec_bruteforce.py) as well, for every search and both classes (bytes; code points with 1- to 4-byte
characters).  The limits that would take gigabytes to reach (WINDOW_BYTES, HOST_CHUNK_BYTES) are patched small; the
lean path's are not (its buffers are sized once from them), so its real boundaries are tested."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, MatchKind, matcher  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, SPEC_BYTES, forced, make_ac  # noqa: E402
from .spec_bruteforce import spec_find  # noqa: E402

AC = matcher._Automaton
SMALL = AC.SMALL_CALL_BYTES      # 256 KiB
ROWS = AC.SMALL_CALL_ROWS        # rows fetched with the status words
LEAN_CAP = 4096                  # rows of the lean workspace
CLASSES = [False, True]
CLASS_IDS = ["bytes", "codepoints"]

# The lean path's patterns.  PLANT goes into filler that holds no "q", "z" or "a": a haystack with k plants has
# exactly k matches in every search.
LEAN_B = [p.encode() for p in ["q€", "𝄞z", "ab"]]
PLANT = "q€".encode()
FILL = [c.encode() for c in ["-", "y", "b", "€", "ß", "☃", "𝄞"]]
# The other tests' patterns: nested and overlapping ones, so that the four searches give four different lists.
PATS_B = [p.encode() for p in ["ab", "abc", "bc", "c", "q€", "ß☃", "𝄞"]]
ALPHA = [c.encode() for c in ["a", "b", "c", "-", " ", "q", "€", "ß", "☃", "𝄞"]]
NESTED_B = [b"a" * i for i in range(1, 17)]


def text(rng, nbytes, alphabet=ALPHA, p=None):
    """Valid UTF-8 of exactly `nbytes` bytes drawn from `alphabet` (padded with "-" after the last whole character)."""
    raw = b"".join(alphabet[i] for i in rng.choice(len(alphabet), size=nbytes, p=p))
    cut = min(nbytes, len(raw))
    while cut < len(raw) and (raw[cut] & 0xC0) == 0x80:
        cut -= 1
    return raw[:cut] + b"-" * (nbytes - cut)


def planted(rng, k, nbytes=None):
    """Filler with PLANT at k places.  `nbytes`: the exact length, with the last plant at the very end."""
    if nbytes is None:
        gaps = rng.integers(0, 9, size=k + 1)
    elif k == 0:
        gaps = [nbytes]
    else:   # k gaps of filler before the plants, none after the last
        free = nbytes - k * len(PLANT)
        gaps = np.diff(np.concatenate([[0], np.sort(rng.integers(0, free + 1, size=k - 1)), [free, free]]))
    out = [text(rng, int(gaps[0]), FILL)]
    for g in gaps[1:]:
        out += [PLANT, text(rng, int(g), FILL)]
    hay = b"".join(out)
    assert nbytes is None or len(hay) == nbytes
    return hay


_ORACLES = {}


def oracle(pats_b, kind):
    key = (tuple(pats_b), kind)
    if key not in _ORACLES:
        _ORACLES[key] = Oracle(pats_b, kind.name)
    return _ORACLES[key]


def expected(pats_b, kind, hay, overlapping, codepoints):
    """The oracle's list for one haystack (bytes) -- code point indexes for the str class; a small haystack with a short
    list is also checked against the brute-force statement."""
    orc = oracle(pats_b, kind)
    got = orc.find_str(hay.decode(), overlapping) if codepoints else orc.find(hay, overlapping)
    if len(hay) <= SPEC_BYTES and len(got) <= 128:
        pats = [p.decode() for p in pats_b] if codepoints else pats_b
        assert got == spec_find(pats, hay.decode() if codepoints else hay, kind.name, overlapping)
    return got


def automata(pats_b, kind, codepoints):
    """The automaton under test and, for the str class, one that keeps no patterns (its find_matches_as_strings slices
    the haystack)."""
    ac = make_ac(pats_b, kind, codepoints)
    plain = AhoCorasick([p.decode() for p in pats_b], kind, store_patterns=False) if codepoints else None
    return ac, plain


@pytest.fixture
def lean(monkeypatch):
    """What each _small_call returned, in order: an array (the lean path answered) or None (it handed over)."""
    seen = []
    small_call = AC._small_call

    def spy(self, hay, overlapping, codepoints):
        r = small_call(self, hay, overlapping, codepoints)
        seen.append(r)
        return r

    monkeypatch.setattr(AC, "_small_call", spy)
    return seen


def lean_check(ac, plain, pats_b, kind, overlapping, codepoints, hay, lean, fits):
    """Every single-haystack list call on `hay` equals the oracle; each one took the lean path (and it answered iff
    `fits`), or, above SMALL_CALL_BYTES, never tried it.  -> the expected list."""
    exp = expected(pats_b, kind, hay, overlapping, codepoints)
    h = hay.decode() if codepoints else hay
    del lean[:]
    assert ac.find_matches_as_indexes(h, overlapping) == exp
    assert ac.find_matches_as_indexes_batch([h], overlapping) == [exp]
    acs = [ac]
    if codepoints:
        want = [h[s:e] for _, s, e in exp]
        assert ac.find_matches_as_strings(h, overlapping) == want
        assert plain.find_matches_as_strings(h, overlapping) == want
        acs.append(plain)
    if len(hay) > SMALL:
        assert lean == []
    else:
        assert [r is not None for r in lean] == [fits] * (2 * len(acs))
        for a in acs:
            assert a._ac._small[torch.cuda.current_device()]["ws"]["capacity"] == LEAN_CAP
    return exp


# ---------------------------------------------------------------- the lean one-haystack path
@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_lean_path_row_counts(search, codepoints, lean):
    """0 and 1 row, the rows that come with the status words and one more, a full lean workspace and one more."""
    kind, overlapping = search
    rng = np.random.default_rng(11)
    ac, plain = automata(LEAN_B, kind, codepoints)
    for k in (0, 1, ROWS, ROWS + 1, LEAN_CAP, LEAN_CAP + 1):
        exp = lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, planted(rng, k), lean, k <= LEAN_CAP)
        assert len(exp) == k


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_lean_path_haystack_sizes(search, codepoints, lean):
    """Empty, one byte, and SMALL_CALL_BYTES - 1, + 0 and + 1 with a match at the very end (above the limit the
    general path scans).  At SMALL_CALL_BYTES + 1 the last character, a 3-byte one, straddles the limit."""
    kind, overlapping = search
    rng = np.random.default_rng(12)
    ac, plain = automata(LEAN_B, kind, codepoints)
    for nbytes in (0, 1, SMALL - 1, SMALL, SMALL + 1):
        hay = planted(rng, 3 if nbytes > 16 else 0, nbytes)
        if nbytes == SMALL + 1:
            assert (hay[SMALL] & 0xC0) == 0x80 and (hay[SMALL - 2] & 0xC0) == 0xC0
        exp = lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, hay, lean, True)
        assert len(exp) == (3 if nbytes > 16 else 0)


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_lean_path_sequences_on_one_automaton(search, codepoints, lean):
    """Calls that leave the lean workspace in every state the next one could trip over, each checked on its own."""
    kind, overlapping = search
    rng = np.random.default_rng(13)
    # a, aa, ..., a x 16 on a run of a: the overlapping list (~16 rows per byte) overflows the lean workspace, while the
    # selected list of every non-overlapping search fits; then one match, then none
    ac, plain = automata(NESTED_B, kind, codepoints)
    run = "ß".encode() + b"a" * 3000 + "☃".encode()
    assert len(oracle(NESTED_B, MatchKind.Standard).find(run, True)) > LEAN_CAP
    exp = lean_check(ac, plain, NESTED_B, kind, overlapping, codepoints, run, lean, False)
    assert overlapping or len(exp) <= LEAN_CAP
    assert len(lean_check(ac, plain, NESTED_B, kind, overlapping, codepoints, "☃-a-ß".encode(), lean, True)) == 1
    assert len(lean_check(ac, plain, NESTED_B, kind, overlapping, codepoints, "☃-ß-𝄞".encode(), lean, True)) == 0
    # a list one row too long for the lean workspace, then one row more than the first copy holds, then exactly that
    ac, plain = automata(LEAN_B, kind, codepoints)
    for k, fits in ((LEAN_CAP + 1, False), (ROWS + 1, True), (ROWS, True), (LEAN_CAP, True), (0, True)):
        assert len(lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, planted(rng, k), lean, fits)) == k
    # 512-byte tasks: the plan of a large haystack outgrows the lean context sized for the default plan (handed over),
    # a small one still fits; then the default plan again
    ac, plain = automata(LEAN_B, kind, codepoints)
    big, small = planted(rng, 50, 200_000), planted(rng, 5, 2000)
    lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, big, lean, True)
    with forced("sieve-small-tasks"):
        lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, big, lean, False)
        lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, small, lean, True)
    lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, big, lean, True)
    lean_check(ac, plain, LEAN_B, kind, overlapping, codepoints, small, lean, True)


# ---------------------------------------------------------------- scan_host's runs
def pack(hays, lead=0):
    """(data, offsets) of a batch whose first haystack starts `lead` bytes into the buffer; the bytes before it and after
    the last one would match if they were scanned."""
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    junk = b"abcq\xe2\x82\xac" * (lead // 6 + 2)
    data = np.frombuffer(junk[:lead] + b"".join(hays) + junk, dtype=np.uint8).copy()
    return data, offs + lead


def runs_of(offs, chunk):
    """The runs [a, b) scan_host cuts a batch into."""
    cuts = [0]
    n = len(offs) - 1
    while cuts[-1] < n:
        h0 = cuts[-1]
        cuts.append(min(max(int(np.searchsorted(offs, offs[h0] + chunk, side="right")) - 1, h0 + 1), n))
    return list(zip(cuts[:-1], cuts[1:]))


def host_input(data, how):
    if how == "numpy":
        return data.copy()
    if how == "readonly":
        a = data.copy()
        a.flags.writeable = False
        return a
    if how == "pinned":
        return torch.from_numpy(data.copy()).pin_memory()
    return torch.from_numpy(data.copy())


def check_scan_host(ac, pats_b, kind, overlapping, codepoints, data, offs, rows_dtype=np.uint32, **kw):
    """scan_host on (data, offs) equals the oracle row for row (haystack ids included) and offset for offset; the
    haystacks in the first SPEC_BYTES with short lists also equal the brute-force statement."""
    lo, hi = int(offs[0]), int(offs[-1])
    raw = np.ascontiguousarray(data[lo:hi]) if isinstance(data, np.ndarray) else data[lo:hi].numpy()
    _, counts, rec = oracle(pats_b, kind).scan_batch(raw, offs - lo, overlapping=overlapping, codepoints=codepoints)
    m, mo = ac.scan_host(data, offs, overlapping, **kw)
    assert m.dtype == rows_dtype and np.array_equal(m, rec.astype(rows_dtype))
    assert mo.dtype == np.int64 and mo[0] == 0 and np.array_equal(np.diff(mo), counts.astype(np.int64))
    seen = 0
    for h in range(len(offs) - 1):
        seen += int(offs[h + 1] - offs[h])
        if seen > SPEC_BYTES:
            break
        if mo[h + 1] - mo[h] > 128:
            continue
        hay = raw[offs[h] - lo:offs[h + 1] - lo].tobytes()
        pats = [p.decode() for p in pats_b] if codepoints else pats_b
        got = [tuple(r) for r in m[mo[h]:mo[h + 1], 1:].tolist()]
        assert got == spec_find(pats, hay.decode() if codepoints else hay, kind.name, overlapping), h
    return m, mo


@pytest.mark.parametrize("chunk, how", [(4 << 10, "numpy"), (16 << 10, "readonly"), (64 << 10, "tensor"), (1 << 20, "pinned")])
@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_scan_host_ragged_runs(search, codepoints, chunk, how):
    """About 2 000 ragged haystacks in runs of `chunk` bytes, offsets that do not start at 0: empty haystacks at run
    boundaries, two haystacks larger than a run (runs of one), the second followed only by empty ones (a last run
    of no bytes)."""
    kind, overlapping = search
    rng = np.random.default_rng(21 + chunk)
    hays = [text(rng, int(n)) if i % 11 else b"" for i, n in enumerate(rng.integers(0, 300, size=1000))]
    hays += [b"", text(rng, chunk * 3 // 2), b""]
    hays += [text(rng, int(n)) if i % 7 else b"" for i, n in enumerate(rng.integers(0, 300, size=1000))]
    hays += [text(rng, chunk * 3 // 2)] + [b""] * 5
    data, offs = pack(hays, lead=1001)
    runs = runs_of(offs, chunk)
    assert len(runs) >= 4 and runs[-1][0] == len(hays) - 5 and offs[-1] == offs[-6]
    assert sum(1 for a, b in runs if b - a == 1) >= 2
    assert any(len(hays[b - 1]) == 0 or len(hays[a]) == 0 for a, b in runs[:-1])
    ac = make_ac(PATS_B, kind, codepoints)
    check_scan_host(ac, PATS_B, kind, overlapping, codepoints, host_input(data, how), offs, chunk_bytes=chunk)


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_scan_host_runs_that_overflow_their_workspace(search, codepoints, monkeypatch):
    """Dense matches: every run's list overflows the run's first workspace (max(4096, 2 x haystacks)), so every run
    is scanned again with room for it, and its rows are rebased to the batch -- directly and through
    find_matches_as_indexes_batch."""
    kind, overlapping = search
    rng = np.random.default_rng(31)
    pats_b = [p.encode() for p in ["a", "aa", "ab", "b", "ßa"]]
    abc = [c.encode() for c in ["a", "b", "ß", "𝄞"]]
    hays = [text(rng, int(n), abc, p=[0.85, 0.05, 0.05, 0.05]) if i % 9 else b"" for i, n in enumerate(rng.integers(0, 3000, size=240))]
    data, offs = pack(hays, lead=3)
    chunk = 64 << 10
    runs = runs_of(offs, chunk)
    _, counts, _ = oracle(pats_b, kind).scan_batch(data[3:], offs - 3, overlapping=overlapping)
    assert len(runs) >= 5 and all(int(counts[a:b].sum()) > 4096 for a, b in runs[:-1])
    ac = make_ac(pats_b, kind, codepoints)
    check_scan_host(ac, pats_b, kind, overlapping, codepoints, data, offs, chunk_bytes=chunk)
    monkeypatch.setattr(AC, "HOST_CHUNK_BYTES", chunk)
    hs = [h.decode() for h in hays] if codepoints else hays
    assert ac.find_matches_as_indexes_batch(hs, overlapping) == [expected(pats_b, kind, h, overlapping, codepoints) for h in hays]


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_batch_calls_in_runs(search, codepoints, monkeypatch):
    """find_matches_as_indexes_batch above HOST_CHUNK_BYTES goes through scan_host's runs."""
    kind, overlapping = search
    rng = np.random.default_rng(41)
    monkeypatch.setattr(AC, "HOST_CHUNK_BYTES", 4 << 10)
    hays = [text(rng, int(n)) if i % 5 else b"" for i, n in enumerate(rng.integers(0, 100, size=1500))]
    hays.insert(700, text(rng, 20_000))
    assert len(runs_of(pack(hays)[1], 4 << 10)) > 10
    ac = make_ac(PATS_B, kind, codepoints)
    hs = [h.decode() for h in hays] if codepoints else hays
    assert ac.find_matches_as_indexes_batch(hs, overlapping) == [expected(PATS_B, kind, h, overlapping, codepoints) for h in hays]


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_scan_host_runs_above_the_window_limit(search, codepoints, monkeypatch):
    """chunk_bytes above WINDOW_BYTES: the runs are scanned one kernel call each without waiting, which has no window
    path, so they must be cut at WINDOW_BYTES.  A haystack above WINDOW_BYTES in a batch that would go in runs takes
    the window path: int64 rows."""
    kind, overlapping = search
    rng = np.random.default_rng(51)
    monkeypatch.setattr(AC, "WINDOW_BYTES", 50_000)
    hays = [text(rng, 1024) for _ in range(1000)]
    ac = make_ac(PATS_B, kind, codepoints)
    data, offs = pack(hays)
    check_scan_host(ac, PATS_B, kind, overlapping, codepoints, data, offs, chunk_bytes=200_000)
    data, offs = pack(hays[:300] + [text(rng, 120_000)] + hays[300:600], lead=5)
    check_scan_host(ac, PATS_B, kind, overlapping, codepoints, data, offs, rows_dtype=np.int64, chunk_bytes=200_000)


# ---------------------------------------------------------------- the host batches and the staging buffer
def batch_calls(ac, hs, overlapping):
    """Every host-batch call on one batch, count_matches_batch first: it starts from the staging buffer as the previous
    batch's calls left it."""
    return {"count": ac.count_matches_batch(hs, overlapping),
            "by_pattern": ac.count_matches_by_pattern_batch(hs, overlapping),
            "patterns": ac.matching_patterns_batch(hs, overlapping),
            "any": ac.is_match_batch(hs),
            "first": ac.find_first_batch(hs)}


def batch_expected(pats_b, kind, hays, overlapping, codepoints):
    """What batch_calls must return, from the oracle's list of each haystack (find_first: element 0 of the
    non-overlapping list, which for Standard is also that of the overlapping one)."""
    lists = [expected(pats_b, kind, h, overlapping, codepoints) for h in hays]
    firsts = [expected(pats_b, kind, h, False, codepoints) for h in hays] if overlapping else lists
    pids = np.array([p for lst in lists for p, _, _ in lst], dtype=np.int64)
    return {"count": [len(lst) for lst in lists],
            "by_pattern": np.bincount(pids, minlength=len(pats_b)).tolist(),
            "patterns": [sorted({p for p, _, _ in lst}) for lst in lists],
            "any": [len(lst) > 0 for lst in lists],
            "first": [lst[0] if lst else None for lst in firsts]}, lists


def check_single_calls(ac, pats_b, h, exp_list, first, overlapping):
    assert ac.is_match(h) == bool(exp_list)
    assert ac.find_first(h) == first
    assert ac.count_matches(h, overlapping) == len(exp_list)
    assert ac.count_matches_by_pattern(h, overlapping) == np.bincount(np.array([p for p, _, _ in exp_list], dtype=np.int64),
                                                                      minlength=len(pats_b)).tolist()
    assert ac.matching_patterns(h, overlapping) == sorted({p for p, _, _ in exp_list})


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_host_batches_sizes_and_stale_staging(search, codepoints):
    """n = 0, 1, 62, 63 (the bytes start exactly at offset 512), 64, 65 (they move to 1024) and 1 000, each small
    batch right after a large one: the staging buffer then holds the large batch's offsets and bytes past the small
    batch's end.  A small batch is short haystacks and a long last one with matches up to its end."""
    kind, overlapping = search
    rng = np.random.default_rng(61)
    enc = (lambda hs: [h.decode() for h in hs]) if codepoints else (lambda hs: hs)
    large = [text(rng, int(n)) for n in rng.integers(10, 21, size=70)] + [text(rng, int(n)) for n in rng.integers(60, 141, size=930)]
    ac = make_ac(PATS_B, kind, codepoints)
    exp_large, _ = batch_expected(PATS_B, kind, large, overlapping, codepoints)
    ac.is_match_batch(enc(large))   # the staging buffer grows to the large batch
    assert ac._ac._staging.numel() >= 8192 + sum(len(h) for h in large) > 1 << 16
    assert batch_calls(ac, enc(large), overlapping) == exp_large
    for n in (1, 62, 63, 64, 65, 0):
        small = [text(rng, int(k)) for k in rng.integers(0, 9, size=max(n - 1, 0))] + ([text(rng, 3000) + b"abc"] if n else [])
        exp, lists = batch_expected(PATS_B, kind, small, overlapping, codepoints)
        assert batch_calls(ac, enc(small), overlapping) == exp, n
        if n:
            assert exp["count"][-1] > 0
            firsts = exp["first"]
            for i in (0, n - 1):
                check_single_calls(ac, PATS_B, enc(small)[i], lists[i], firsts[i], overlapping)
        assert batch_calls(ac, enc(large), overlapping) == exp_large, n


@pytest.mark.parametrize("codepoints", CLASSES, ids=CLASS_IDS)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_host_batches_of_empty_haystacks(search, codepoints):
    """Batches of empty haystacks only (no bytes at all), after a call that filled the staging buffer."""
    kind, overlapping = search
    rng = np.random.default_rng(71)
    ac = make_ac(PATS_B, kind, codepoints)
    full = [text(rng, 200) for _ in range(500)]
    ac.count_matches_batch([h.decode() for h in full] if codepoints else full, overlapping)
    e = "" if codepoints else b""
    for n in (0, 1, 63, 64, 1000):
        assert batch_calls(ac, [e] * n, overlapping) == {"count": [0] * n, "by_pattern": [0] * len(PATS_B), "patterns": [[]] * n,
                                                         "any": [False] * n, "first": [None] * n}, n
    check_single_calls(ac, PATS_B, e, [], None, overlapping)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_host_calls_take_any_u8_buffer(search):
    """bytes, bytearray, memoryview and uint8 / int8 numpy arrays, mixed in one batch and one by one, through every
    host call; 2-D and non-contiguous buffers raise TypeError."""
    kind, overlapping = search
    rng = np.random.default_rng(81)
    hays = [text(rng, int(n)) for n in rng.integers(0, 400, size=40)]
    forms = [bytes, bytearray, lambda h: memoryview(h), lambda h: np.frombuffer(h, dtype=np.uint8),
             lambda h: np.frombuffer(h, dtype=np.int8)]
    bufs = [forms[i % len(forms)](h) for i, h in enumerate(hays)]
    ac = make_ac(PATS_B, kind)
    exp, lists = batch_expected(PATS_B, kind, hays, overlapping, False)
    assert batch_calls(ac, bufs, overlapping) == exp
    assert ac.find_matches_as_indexes_batch(bufs, overlapping) == lists
    for i, b in enumerate(bufs[:10]):
        assert ac.find_matches_as_indexes(b, overlapping) == lists[i]
        check_single_calls(ac, PATS_B, b, lists[i], exp["first"][i], overlapping)
    bad = [np.zeros((2, 4), dtype=np.uint8), memoryview(bytearray(b"abcabcab"))[::2], np.frombuffer(b"abcabcab", dtype=np.uint8)[::2]]
    for b in bad:
        for call in (lambda: ac.find_matches_as_indexes(b, overlapping), lambda: ac.find_matches_as_indexes_batch([b"ab", b], overlapping),
                     lambda: ac.is_match(b), lambda: ac.is_match_batch([b"ab", b]), lambda: ac.find_first(b),
                     lambda: ac.find_first_batch([b]), lambda: ac.count_matches(b, overlapping),
                     lambda: ac.count_matches_batch([b"ab", b], overlapping), lambda: ac.count_matches_by_pattern(b, overlapping),
                     lambda: ac.count_matches_by_pattern_batch([b], overlapping), lambda: ac.matching_patterns(b, overlapping),
                     lambda: ac.matching_patterns_batch([b"ab", b], overlapping)):
            with pytest.raises(TypeError):
                call()
