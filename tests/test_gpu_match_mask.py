"""GPU tests of the match mask (-m gpu): match_mask_device, match_spans and match_spans_batch of the three classes.
Every mask is compared with the union of the oracle's record spans, and with the difference-array mask built from
scan_device's own rows (+1 at every start, -1 at every end, a prefix sum, > 0).  Covered: every search on the sieve
(cover mode and mask epilogue), the sieve with 512-byte tasks and the staged table walker (rows path); str, bytes and
token ids of every width; the cover mode, filtered and not, at the sieve geometries of test_gpu_sieve_geometry.py;
pattern sets against subset_scan_batch; stretches around ACB_LONG_STRETCH and the workspace retry; haystacks of 0-70
bytes packed back to back with offsets[0] > 0; the run and window paths with a small WINDOW_BYTES at unaligned starts,
and one haystack above 2 GiB; and two threads sharing one automaton."""
import random
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200.matcher import _encode_host_tokens  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, dev, dev_at, forced, make_ac  # noqa: E402
from .sieve_geometry_helpers import assert_geometry, case_inputs, fanout, geometry, planted, subset_scan_batch  # noqa: E402
from .sieve_inputs import FANOUTS  # noqa: E402

ENGINES = ("sieve", "sieve-small-tasks", "staged")


def union_mask(rec, offs, total):
    """Bytes covered by records (haystack, pattern, start, end), haystack-relative byte offsets."""
    d = np.zeros(total + 1, dtype=np.int64)
    if len(rec):
        base = np.asarray(offs, dtype=np.int64)[rec[:, 0].astype(np.int64)]
        np.add.at(d, base + rec[:, 2].astype(np.int64), 1)
        np.add.at(d, base + rec[:, 3].astype(np.int64), -1)
    return np.cumsum(d[:total]) > 0


def oracle_mask(pats, kind, data, offs, overlapping):
    _, _, rec = Oracle(pats, kind.name).scan_batch(data, offs, overlapping=overlapping)
    return union_mask(rec, offs, len(data))


def diff_mask(ac, d, o, overlapping, **kw):
    """What a user builds without the feature: scan_device's byte rows, index_add_, cumsum, > 0 (on the device)."""
    m, _, _ = ac._ac.scan_device(d, o, overlapping, False, **kw)
    m = m.long()
    base = o[m[:, 0]]
    acc = torch.zeros(d.numel() + 1, dtype=torch.int64, device=d.device)
    acc.index_add_(0, base + m[:, 2], torch.ones_like(base))
    acc.index_add_(0, base + m[:, 3], -torch.ones_like(base))
    return (torch.cumsum(acc[:-1], 0) > 0).cpu().numpy()


def packed_batch(seed, utf8=False, first=37):
    """Haystacks of 0-70 bytes back to back after `first` bytes of lead-in, with occurrences at both ends of most."""
    rng = random.Random(seed)
    alpha = ["a", "b", "c", "é", "€"] if utf8 else ["a", "b", "c"]
    pats = ["".join(rng.choice(alpha) for _ in range(rng.randint(1, 5))) for _ in range(12)]
    pats += [pats[0], "abcab", "bcab", "cab", "ab", "c"]   # a duplicate, a nested family
    hays = []
    for i in range(120):
        n = rng.randint(0, 70) if i % 9 else i % 3
        s = "".join(rng.choice(alpha) for _ in range(n))
        if n > 8 and i % 2:
            s = rng.choice(pats) + s + rng.choice(pats)
        hays.append(s)
    lead = b"abcab" * (first // 5 + 1)
    enc = [h.encode() for h in hays]
    data = np.frombuffer(lead[:first] + b"".join(enc), dtype=np.uint8).copy()
    offs = np.concatenate([[first], first + np.cumsum([len(e) for e in enc])]).astype(np.int64)
    return [p.encode() for p in pats], data, offs


def check_mask(ac, pats, kind, data, offs, overlapping, shift=0, flt_args=None):
    d, o = dev_at(data, shift), dev(offs)
    got = ac.match_mask_device(d, o, overlapping, **(flt_args or {})).cpu().numpy()
    assert got.shape == (len(data),) and got.dtype == bool
    want = oracle_mask(pats, kind, data, offs, overlapping)
    assert np.array_equal(got, want), (kind, overlapping, np.flatnonzero(got != want)[:10])
    assert not got[:int(offs[0])].any()
    return d, o, got


# ---------------------------------------------------------------- every search on every engine, str and bytes
@pytest.mark.parametrize("utf8", [False, True], ids=["bytes", "str"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_searches_on_engines(search, engine, utf8):
    kind, overlapping = search
    for seed in range(3):
        pats, data, offs = packed_batch(seed, utf8)
        with forced(engine):
            ac = make_ac(pats, kind, utf8)
            d, o, got = check_mask(ac, pats, kind, data, offs, overlapping, shift=seed * 255)
            st = ac._ac.last_stats
            assert st["mode"] == "match_mask" and st["engine"] == ("table" if engine == "staged" else "sieve"), st
            if engine != "staged" and not overlapping:
                assert st["list_records"] > 0 and "long_stretches" in st
            assert np.array_equal(got, diff_mask(ac, d, o, overlapping))


@pytest.mark.parametrize("width", [torch.uint16, torch.int32, torch.int64], ids=["u16", "i32", "i64"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_token_ids(search, width):
    kind, overlapping = search
    rng = np.random.default_rng(7)
    pats = [rng.integers(0, 40, size=rng.integers(1, 4)).tolist() for _ in range(20)] + [[1, 2, 3], [2, 3], [3], [65535]]
    lens = rng.integers(0, 60, size=50)
    ids = rng.integers(0, 40, size=int(lens.sum()))
    ids[::17] = 65535
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    tac = TokenAhoCorasick(pats, kind)
    got = tac.match_mask_device(torch.from_numpy(ids.astype(np.int64)).to(width).cuda(), dev(offs), overlapping).cpu().numpy()
    enc = _encode_host_tokens(ids, "ids")
    pb = [_encode_host_tokens(p, "p").tobytes() for p in pats]
    want = oracle_mask(pb, kind, enc, offs * 3, overlapping)[::3]
    assert got.shape == (len(ids),) and np.array_equal(got, want)
    hays = [ids[offs[h]:offs[h + 1]].tolist() for h in range(len(lens))]
    spans = tac.match_spans_batch(hays, overlapping)
    assert spans == [runs(want[offs[h]:offs[h + 1]]) for h in range(len(lens))]
    assert tac.match_spans(hays[3], overlapping) == spans[3]


def runs(bits):
    out, p = [], 0
    bits = list(bits)
    while p < len(bits):
        if bits[p]:
            q = p
            while q < len(bits) and bits[q]:
                q += 1
            out.append((p, q))
            p = q
        else:
            p += 1
    return out


# ---------------------------------------------------------------- the host forms
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_match_spans(search):
    kind, overlapping = search
    pats, data, offs = packed_batch(11, utf8=True)
    hays = [data[offs[h]:offs[h + 1]].tobytes().decode() for h in range(len(offs) - 1)]
    sac = AhoCorasick([p.decode() for p in pats], kind)
    bac = BytesAhoCorasick(pats, kind)
    for ac, hs in ((sac, hays), (bac, [h.encode() for h in hays])):
        got = ac.match_spans_batch(hs, overlapping)
        for h, hay in enumerate(hs):
            cov = np.zeros(len(hay), dtype=bool)
            for _, s, e in ac.find_matches_as_indexes(hay, overlapping):
                cov[s:e] = True
            assert got[h] == runs(cov), h
        assert ac.match_spans(hs[5], overlapping) == got[5]
    # patterns=: the subset's spans
    sets = [[p for p in range(len(pats)) if (p + h) % 3] for h in range(len(hays))]
    got = bac.match_spans_batch([h.encode() for h in hays], overlapping, patterns=sets)
    for h, hay in enumerate(hays):
        cov = np.zeros(len(hay.encode()), dtype=bool)
        for _, s, e in bac.find_matches_as_indexes(hay.encode(), overlapping, patterns=sets[h]):
            cov[s:e] = True
        assert got[h] == runs(cov), h
    assert sac.match_spans("", overlapping) == [] and sac.match_spans_batch([], overlapping) == []


# ---------------------------------------------------------------- the cover mode at the sieve geometries
RINGS = (1, 8)
DEFAULT_TASK = 16384


def check_cover(pats, data, offs, want, shift, utf8=False):
    """The cover mode, unfiltered and with pattern sets ("all", a seeded 30 %, and an index past the sets), and the
    mask epilogue of LeftmostLongest, each against the oracle, with the geometry asserted."""
    ac = make_ac(pats, MatchKind.Standard, utf8)
    check_mask(ac, pats, MatchKind.Standard, data, offs, True, shift)
    assert_geometry(ac, want)
    n = len(offs) - 1
    rng = np.random.default_rng(len(pats))
    sets = [list(range(len(pats))), [p for p in range(len(pats)) if rng.random() < 0.3]]
    idx = rng.integers(0, 2, size=n)
    idx[::7] = 2
    ps = ac.pattern_sets(sets)
    d, o = dev_at(data, shift), dev(offs)
    words = ac._ac.mask_device(d, o, True, flt=(ps, torch.from_numpy(idx).cuda()))
    got = ac._ac.unpack_mask(words, len(data)).cpu().numpy()
    assert_geometry(ac, want)
    assert ac._ac.last_stats["pattern_sets"] == 2
    _, _, rec = subset_scan_batch(pats, "Standard", data, offs, sets, idx, overlapping=True)
    assert np.array_equal(got, union_mask(rec, offs, len(data)))
    ll = make_ac(pats, MatchKind.LeftmostLongest, utf8)
    check_mask(ll, pats, MatchKind.LeftmostLongest, data, offs, False, shift)
    assert_geometry(ll, want)


@pytest.mark.parametrize("ring", RINGS)
@pytest.mark.parametrize("w", range(1, 9))
def test_cover_window_by_ring(monkeypatch, w, ring):
    pats, data, offs = planted(False)
    with geometry(monkeypatch, w, ring, DEFAULT_TASK):
        check_cover(pats, data, offs, {"window": w, "ring": ring, "task_bytes": DEFAULT_TASK}, shift=(0, 1, 511)[(w + ring) % 3])


@pytest.mark.parametrize("w", (1, 4, 5, 8))
def test_cover_small_tasks(monkeypatch, w):
    pats, data, offs = planted(False)
    with geometry(monkeypatch, w, 8, 512):
        check_cover(pats, data, offs, {"window": w, "ring": 8, "task_bytes": 512}, shift=w % 2)


@pytest.mark.parametrize("w", (1, 5, 8))
def test_cover_code_points(monkeypatch, w):
    pats, data, offs = planted(True)
    with geometry(monkeypatch, w, 4, DEFAULT_TASK):
        check_cover(pats, data, offs, {"window": w, "ring": 4, "task_bytes": DEFAULT_TASK}, shift=1, utf8=True)


@pytest.mark.parametrize("task_bytes", (DEFAULT_TASK, 512))
@pytest.mark.parametrize("budget", ["default", "shallow", "saturated"])
def test_cover_filter_budget(monkeypatch, budget, task_bytes):
    name, nbytes = {"default": ("planted", None), "shallow": ("decoys", 8192), "saturated": ("dense", 4096)}[budget]
    pats, data, offs = case_inputs((name, False))
    want = {"window": 5, "task_bytes": task_bytes}
    if nbytes == 4096:
        want["bloom_bytes"] = 4096
    with geometry(monkeypatch, 5, 1, task_bytes, nbytes):
        check_cover(pats, data, offs, want, shift=task_bytes // 512 % 3)


@pytest.mark.parametrize("w", (1, 8))
@pytest.mark.parametrize("fan", FANOUTS)
def test_cover_trie_fanout(monkeypatch, fan, w):
    pats, data, offs = fanout(fan)
    with geometry(monkeypatch, w, 8, DEFAULT_TASK):
        check_cover(pats, data, offs, {"window": w, "ring": 8, "task_bytes": DEFAULT_TASK}, shift=w % 3)


# ---------------------------------------------------------------- pattern sets
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_pattern_sets(search):
    kind, overlapping = search
    pats, data, offs = packed_batch(5)
    n = len(offs) - 1
    ac = BytesAhoCorasick(pats, kind)
    rng = np.random.default_rng(3)
    sets = [list(range(len(pats))), [], [0, len(pats) - 2, len(pats) - 1]] + [[p for p in range(len(pats)) if rng.random() < 0.3]]
    ps = ac.pattern_sets(sets)
    idx = rng.integers(0, len(sets), size=n)
    d, o = dev_at(data, 3), dev(offs)
    got = ac.match_mask_device(d, o, overlapping, pattern_sets=ps, set_index=torch.from_numpy(idx).cuda()).cpu().numpy()
    assert ac._ac.last_stats["pattern_sets"] == len(sets) and ac._ac.last_stats["engine"] == "sieve"
    _, _, rec = subset_scan_batch(pats, kind, data, offs, sets, idx, overlapping)
    assert np.array_equal(got, union_mask(rec, offs, len(data)))
    # the "all" set is the unfiltered call; an index outside [0, n_sets) (int32 and int64) admits nothing
    got_all = ac.match_mask_device(d, o, overlapping, pattern_sets=ps, set_index=torch.zeros(n, dtype=torch.int64, device="cuda"))
    assert torch.equal(got_all, ac.match_mask_device(d, o, overlapping))
    for dt, bad in ((torch.int32, -1), (torch.int32, len(sets)), (torch.int64, 1 << 40)):
        words = ac._ac.mask_device(d, o, overlapping, flt=(ps, torch.full((n,), bad, dtype=dt, device="cuda")))
        assert not ac._ac.unpack_mask(words, len(data)).any()


# ---------------------------------------------------------------- long stretches and the workspace retry
@pytest.mark.parametrize("kind", [MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_long_stretches_and_retry(kind):
    """[aa] over a * m: m - 1 overlapping records, every other one selected, so an odd m leaves the last byte
    uncovered.  The records straddle ACB_LONG_STRETCH; a fresh automaton's first workspace holds 1 024 records."""
    L = _capi.ACB_LONG_STRETCH
    for m in (L, L + 1, L + 2, 2 * L + 1):
        data = np.frombuffer(b"xy" + b"a" * m + b"b" * 5 + b"a" * 7, dtype=np.uint8).copy()
        offs = np.array([2, 2 + m, len(data)], dtype=np.int64)
        ac = BytesAhoCorasick([b"aa", b"bab"], kind)
        with forced("sieve"):
            words = ac._ac.mask_device(dev(data), dev(offs), False, capacity=1)
        got = ac._ac.unpack_mask(words, len(data)).cpu().numpy()
        assert np.array_equal(got, oracle_mask([b"aa", b"bab"], kind, data, offs, False)), m
        assert got[2 + m - 1] == (m % 2 == 0)
        st = ac._ac.last_stats
        assert st["long_stretches"] == (1 if m - 1 > L else 0) and st["list_records"] == m - 1 + 6, st
        assert ac._ac._ws[(torch.cuda.current_device(), 0)]["capacity"] > 1024


# ---------------------------------------------------------------- runs and windows
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_run_and_window_paths(monkeypatch, search):
    """WINDOW_BYTES = 1 000 + 13: runs of whole haystacks and windows of larger ones start at unaligned bits."""
    kind, overlapping = search
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 1013)
    rng = random.Random(9)
    pats = [b"abc", b"bca", b"cab", b"abcabcab", b"c", b"aa"]
    hays = [bytes(rng.choice(b"abcx") for _ in range(n)) for n in (5, 700, 400, 3000, 1, 0, 2500, 90, 1013, 1014)]
    lead = 29
    data = np.frombuffer(b"q" * lead + b"".join(hays), dtype=np.uint8).copy()
    offs = np.concatenate([[lead], lead + np.cumsum([len(h) for h in hays])]).astype(np.int64)
    for engine in ("sieve", "staged"):
        with forced(engine):
            ac = BytesAhoCorasick(pats, kind)
            check_mask(ac, pats, kind, data, offs, overlapping, shift=5)
            assert ac._ac.last_stats["windows"] is True


def test_haystack_above_2_gib():
    """One real haystack past 2^31 bytes (windows of WINDOW_BYTES sharing max_pattern_len - 1 bytes), both searches:
    occurrences at the start, inside the first window only, across its end (so inside the second window only), past
    it, and at the end."""
    size = (1 << 31) + 4099
    data = torch.zeros(size + 11, dtype=torch.uint8, device="cuda")
    hay = data[11:]
    pat = b"needle-in-a-haystack"
    wb = matcher._Automaton.WINDOW_BYTES
    starts = [0, wb - 3 * len(pat), wb - 7, wb + 100, size - len(pat)]   # (apart: no placement overwrites another)
    for s in starts:
        hay[s:s + len(pat)] = torch.frombuffer(bytearray(pat), dtype=torch.uint8).cuda()
    want = torch.zeros(size + 11, dtype=torch.bool, device="cuda")
    for s in starts:
        want[11 + s:11 + s + len(pat)] = True
    offs = torch.tensor([11, size + 11], dtype=torch.int64, device="cuda")
    for overlapping in (True, False):
        ac = BytesAhoCorasick([pat, b"haystack"])
        got = ac.match_mask_device(data, offs, overlapping)
        assert torch.equal(got, want), overlapping
        assert ac._ac.last_stats["windows"] is True
        del got
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- threads
def test_two_threads():
    pats, data, offs = packed_batch(21)
    ac = BytesAhoCorasick(pats)
    want = {o: oracle_mask(pats, MatchKind.Standard, data, offs, o) for o in (False, True)}
    errors = []

    def work(overlapping):
        try:
            d, o = dev(data), dev(offs)
            for _ in range(20):
                got = ac.match_mask_device(d, o, overlapping).cpu().numpy()
                assert np.array_equal(got, want[overlapping])
        except Exception as e:   # noqa: BLE001 -- reported below
            errors.append(e)

    ts = [threading.Thread(target=work, args=(o,)) for o in (False, True)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
