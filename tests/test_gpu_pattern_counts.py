"""GPU tests of count_matches_by_pattern (-m gpu): per-pattern match counts over a batch from
acb_pattern_counts_overlapping (the sieve kernel's pattern mode), acb_pattern_counts_non_overlapping (the sieve's list
scan and the pattern epilogue, serial and grid-marked stretches) and the table walkers' composition.  The expected
answer is always the bincount of the oracle's pattern column; every answer is also compared with the bincount of
scan_device's pattern column and its total with count_matches_device's.  Also: stretches around ACB_LONG_STRETCH
records, a hot pattern, large pattern sets, a workspace retry that adds nothing, accumulation, code points, the golden
vectors, runs and windows above one call's range, config 4 at size and two threads."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, Implementation, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402

from .gpu_helpers import KINDS, SEARCH_IDS, SEARCHES, dev, forced  # noqa: E402
from .sieve_geometry_helpers import oracle_hist  # noqa: E402
from .test_gpu_count import ENGINES, KIND_IDS, L_STRETCH, VECTORS, batch, stretch_batch  # noqa: E402


def check(pats, data, offs, kind, overlapping=False, ac=None, capacity=None):
    """count_matches_by_pattern_device equals the oracle's histogram, the bincount of scan_device's pattern column, and
    sums to count_matches_device's total.  -> (ac, last_stats)."""
    exp = oracle_hist(pats, data, offs, kind, overlapping)
    ac = ac or BytesAhoCorasick(pats, kind)
    d, o = dev(data), dev(offs)
    got = ac.count_matches_by_pattern_device(d, o, overlapping) if capacity is None else ac._ac.pattern_counts_device(d, o, overlapping, capacity)
    assert got.dtype == torch.int64 and got.shape == (len(pats),)
    got = got.cpu().numpy()
    stats = dict(ac._ac.last_stats)
    assert stats["mode"] == "pattern_counts"
    assert np.array_equal(got, exp)
    m, _, _ = ac.scan_device(d, o, overlapping)
    assert np.array_equal(np.bincount(m[:, 1].long().cpu().numpy(), minlength=len(pats)), got)
    assert int(ac.count_matches_device(d, o, overlapping).sum().item()) == int(got.sum())
    return ac, stats


# ---------------------------------------------------------------- parity
@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("shortest", [1, 2, 3, 5, 8])
def test_ragged_small_alphabet(variant, search, shortest):
    kind, overlapping = search
    rng = np.random.default_rng(300 + shortest)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 7))).astype(np.uint8)) for _ in range(40)})
    pats += pats[:2]   # duplicates: distinct ids, same bytes
    hays = []
    for i in range(300):
        h = rng.integers(97, 101, size=int(rng.integers(0, 40 * shortest + 1))).astype(np.uint8).tobytes() if i % 19 else b""
        if i % 4 == 0 and h:
            at = int(rng.integers(0, len(h) + 1))
            h = h[:at] + pats[i % len(pats)] * 3 + h[at:]
        hays.append(h)
    data, offs = batch(hays)
    with forced(variant):
        _, st = check(pats, data, offs, kind, overlapping)
        assert st["engine"] == ("table" if variant == "staged" else "sieve")


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_full_byte_range_and_straddling(variant, search):
    kind, overlapping = search
    rng = np.random.default_rng(7)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(2, 5))).astype(np.uint8)) for _ in range(300)]
    pats += [b"\x00\xff", b"\xff\x00\x80", b"\x00", b"abcd", b"\x00"]
    data = rng.integers(1, 256, size=300_000, dtype=np.uint8).astype(np.uint8)
    offs = np.unique(np.concatenate([[0, len(data)], rng.integers(0, len(data), size=2000)])).astype(np.int64)
    data[offs[5:40:3]] = 0
    with forced(variant):
        check(pats, data, offs, kind, overlapping)
        d2, o2 = batch([b"xxab", b"cdxx", b"a", b"bcd", b"abcd", b""] * 40)   # matches across haystacks never count
        check(pats, d2, o2, kind, overlapping)


# ---------------------------------------------------------------- the grid path for long stretches
@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_stretches_around_the_long_stretch_limit(variant, kind):
    rng = np.random.default_rng(5)
    hays, n_long = stretch_batch(rng)
    pats = [b"a", b"aa", b"b"] if kind != MatchKind.LeftmostFirst else [b"aa", b"a", b"b"]
    data, offs = batch(hays)
    with forced(variant):
        ac, st = check(pats, data, offs, kind)
        assert st["long_stretches"] == n_long, st
        for h, want in ((b"a" * (L_STRETCH // 2), 0), (b"a" * (L_STRETCH // 2) + b"b", 0), (b"a" * (L_STRETCH // 2 + 1), 1)):
            d, o = batch([h])
            _, st = check(pats, d, o, kind, ac=ac)
            assert st["long_stretches"] == want


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_dense_single_haystacks_on_the_grid(kind):
    """400 k-record haystacks with nested and self-overlapping patterns (and a duplicate): the marks follow the
    leftmost kinds' look-ahead and restarts, next to short haystacks in the same batch."""
    rng = np.random.default_rng(9)
    pats = [b"ab", b"aba", b"bab", b"abab", b"b", b"baab", b"aa", b"ab"]
    big = rng.choice(list(b"ab"), size=400_000).astype(np.uint8).tobytes()
    hays = [b"abab", big, b"", b"babab" * 10, big[:70_000], b"x"]
    data, offs = batch(hays)
    with forced("sieve"):
        _, st = check(pats, data, offs, kind)
        assert st["long_stretches"] == 2 and st["list_records"] > 300_000


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_hot_pattern(search):
    """One single-byte pattern (twice: two ids) matching every position of 24 MiB plus a few rare ones: every
    verification round adds to the same counters, and the counts stay exact."""
    kind, overlapping = search
    data = np.full(24 << 20, ord("a"), dtype=np.uint8)
    rng = np.random.default_rng(12)
    pos = np.sort(rng.choice(len(data) // 8, size=300, replace=False)) * 8
    for k, p in enumerate(pos):
        data[p:p + 5] = np.frombuffer([b"xqzjk", b"vwxyz"][k % 2], dtype=np.uint8)
    pats = [b"a", b"xqzjk", b"vwxyz", b"zzqzz", b"a"]
    offs = np.array([0, 1 << 20, 13 << 20, len(data)], dtype=np.int64)
    with forced("sieve"):
        check(pats, data, offs, kind, overlapping)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_large_pattern_sets(search):
    """Config 3's 10 k and config 4's 100 k patterns: a histogram far larger than a warp's round."""
    kind, overlapping = search
    pats3, data3, offs3 = W.config3(n_lines=20_000)
    check(pats3, data3, offs3, kind, overlapping)
    pats4, data4 = W.config4(hay_bytes=4 << 20)
    check(pats4, data4, np.array([0, 1 << 20, 3 << 20, len(data4)], dtype=np.int64), kind, overlapping)


# ---------------------------------------------------------------- workspace retry, accumulation
def test_workspace_retry_adds_nothing_on_the_failed_attempt():
    pats = [b"a", b"aa", b"b"]
    data, offs = batch([b"a" * 30_000, b"ab" * 100, b"b" * 5000])
    L = _capi.lib()
    with forced("sieve"):
        for kind in KINDS:
            ac = BytesAhoCorasick(pats, kind)
            n0 = L.acb_launch_count()
            check(pats, data, offs, kind, ac=ac, capacity=1)
            assert L.acb_launch_count() >= n0 + 2
    # a direct call with a workspace too small for the list leaves the counts as they were
    ac = BytesAhoCorasick(pats, MatchKind.LeftmostLongest)
    a = ac._ac
    d, o = dev(data), dev(offs)
    n = len(offs) - 1
    with forced("sieve"), torch.cuda.device(d.device):
        sieve_t, _ = a.sieve(d.device)
        plan = a._plan(d, n)
        ws = a._workspace(d.device, plan, n, 16, 0)
        st = a._ws_struct(ws)
        counts = torch.tensor([7, 8, 9], dtype=torch.int64, device=d.device)
        stream = torch.cuda.current_stream(d.device).cuda_stream
        rc = a._L.acb_pattern_counts_non_overlapping(a._h, sieve_t.data_ptr(), d.data_ptr(), o.data_ptr(), n, d.numel(),
                                                     C.byref(plan), C.byref(st), counts.data_ptr(), stream)
        assert rc == _capi.ACB_OK, _capi.last_error()
        tot = ws["total"].tolist()
        assert tot[1] == 0 and tot[4] > 16
        assert counts.tolist() == [7, 8, 9]


def test_two_abi_calls_add():
    pats = [b"ab", b"b", b"ab"]
    data, offs = batch([b"abab" * 100, b"xbx", b""])
    ac = BytesAhoCorasick(pats)
    a = ac._ac
    d, o = dev(data), dev(offs)
    n = len(offs) - 1
    exp = oracle_hist(pats, data, offs, MatchKind.Standard, True)
    exp_non = oracle_hist(pats, data, offs, MatchKind.Standard, False)
    with forced("sieve"), torch.cuda.device(d.device):
        sieve_t, _ = a.sieve(d.device)
        stream = torch.cuda.current_stream(d.device).cuda_stream
        counts = torch.zeros(3, dtype=torch.int64, device=d.device)
        scratch = torch.empty(3, dtype=torch.int64, device=d.device)
        for _ in range(2):
            assert a._L.acb_pattern_counts_overlapping(a._h, sieve_t.data_ptr(), d.data_ptr(), o.data_ptr(), n, d.numel(),
                                                       counts.data_ptr(), scratch.data_ptr(), stream) == _capi.ACB_OK
        assert np.array_equal(counts.cpu().numpy(), 2 * exp)
        plan = a._plan(d, n)
        ws = a._workspace(d.device, plan, n, 4096, 0)
        st = a._ws_struct(ws)
        for _ in range(2):
            assert a._L.acb_pattern_counts_non_overlapping(a._h, sieve_t.data_ptr(), d.data_ptr(), o.data_ptr(), n, d.numel(),
                                                           C.byref(plan), C.byref(st), counts.data_ptr(), stream) == _capi.ACB_OK
        assert np.array_equal(counts.cpu().numpy(), 2 * exp + 2 * exp_non)
        assert ws["total"].tolist()[:2] == [int(exp_non.sum()), 1]


# ---------------------------------------------------------------- code points, golden vectors
def test_utf8_haystacks_on_the_str_class():
    pats = ["é", "éé", "☃x", "needle", "x", "é"]
    hays = ["", "é" * 500, "☃x" * 40 + "needle", "aé☃xé" * 300, "x" * 10_000, "ascii only"]
    for variant in ENGINES:
        with forced(variant):
            for kind in KINDS:
                ac = AhoCorasick(pats, kind)
                for overlapping in ([False, True] if kind == MatchKind.Standard else [False]):
                    per = [ac.find_matches_as_indexes(h, overlapping) for h in hays]
                    want = np.bincount([m[0] for ms in per for m in ms], minlength=len(pats)).tolist()
                    assert ac.count_matches_by_pattern_batch(hays, overlapping) == want
                    assert ac.count_matches_by_pattern(hays[3], overlapping) == np.bincount([m[0] for m in per[3]], minlength=len(pats)).tolist()
                    data, offs = batch(hays)
                    assert ac.count_matches_by_pattern_device(dev(data), dev(offs), overlapping).cpu().tolist() == want


@pytest.mark.parametrize("variant", ENGINES)
def test_reference_vectors(variant):
    with forced(variant):
        for vec in VECTORS:
            kind = MatchKind[vec["kind"]]
            hay = vec["haystack"]
            ac = AhoCorasick(vec["patterns"], kind) if vec["cls"] == "str" else BytesAhoCorasick([p.encode() for p in vec["patterns"]], kind)
            hay = hay if vec["cls"] == "str" else hay.encode()
            if vec.get("error"):
                with pytest.raises(ValueError):
                    ac.count_matches_by_pattern(hay, overlapping=True)
                continue
            found = ac.find_matches_as_indexes(hay, overlapping=vec["overlapping"])
            want = np.bincount([m[0] for m in found], minlength=len(vec["patterns"])).tolist()
            if "expect_indexes" in vec:
                assert want == np.bincount([m[0] for m in vec["expect_indexes"]], minlength=len(vec["patterns"])).tolist()
            assert ac.count_matches_by_pattern(hay, overlapping=vec["overlapping"]) == want, vec


# ---------------------------------------------------------------- runs and windows above one call's range
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_windows_and_runs(search, monkeypatch):
    kind, overlapping = search
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    data, offs = W.ragged(400, 3000, b"abcdxyz", seed=32)
    exp = oracle_hist(pats, data, offs, kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    assert np.array_equal(ac.count_matches_by_pattern_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
    assert np.array_equal(ac.count_matches_by_pattern_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
    assert ac._ac.last_stats["windows"]


@pytest.mark.parametrize("variant", ["sieve", "staged"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_oversized_haystack_in_windows(variant, search, monkeypatch):
    """One haystack above the window limit among small ones, with matches inside the bytes windows share (counted
    once, per pattern) and a dense stretch; the non-overlapping counts go through the serial selection."""
    kind, overlapping = search
    limit = 30_001
    pats = [b"needle12345", b"needle", b"aa", b"a", b"needle"]
    rng = np.random.default_rng(8)
    big = bytearray(rng.choice(list(b"xa"), size=200_000).astype(np.uint8).tobytes())
    step = limit - (len(pats[0]) - 1)
    for p in (limit - 8, step - 3, 2 * step + 1, 150_000):
        big[p:p + 11] = pats[0]
    hays = [b"xneedle", b"xx", bytes(big), b"needle1", b"aaaa", bytes(b"a" * 70_000) + pats[0]]
    data, offs = batch(hays)
    exp = oracle_hist(pats, data, offs, kind, overlapping)
    exp_big = oracle_hist(pats, np.frombuffer(bytes(big), dtype=np.uint8), np.array([0, len(big)]), kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", limit)
    with forced(variant):
        assert np.array_equal(ac.count_matches_by_pattern_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
        assert ac.count_matches_by_pattern(bytes(big), overlapping) == exp_big.tolist()


def test_config4_single_4gib_haystack_overlapping():
    """BASELINE config 4 at size: ONE haystack of 2^32 bytes, 100k patterns, overlapping, in windows; equal to the
    bincount of scan_device's list."""
    n = 1 << 32
    pats = W.random_lowercase_patterns(100_000, 5, 8, 4)
    g = torch.Generator(device="cuda")
    g.manual_seed(1004)
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    for a in range(0, n, 1 << 28):
        d[a:a + (1 << 28)] = torch.randint(97, 123, (1 << 28,), dtype=torch.uint8, device="cuda", generator=g)
    ac = BytesAhoCorasick(pats, implementation=Implementation.ContiguousNFA)
    o = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    got = ac.count_matches_by_pattern_device(d, o, overlapping=True)
    m, _, total = ac.scan_device(d, o, overlapping=True)
    assert torch.equal(got, torch.bincount(m[:, 1], minlength=len(pats))) and total > 5_000_000
    del d, m


# ---------------------------------------------------------------- threads
def test_two_threads_share_one_automaton():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(2, 7))).astype(np.uint8)) for _ in range(60)})
    ac = BytesAhoCorasick(pats, MatchKind.Standard)
    inputs = []
    for t in range(2):
        data, offs = W.ragged(300, 200 + 100 * t, b"abcdxyz", seed=50 + t)
        hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
        inputs.append((hays, oracle_hist(pats, data, offs, MatchKind.Standard, t == 1).tolist()))
    errors = []

    def work(t):
        try:
            hays, exp = inputs[t]
            for _ in range(25):
                assert ac.count_matches_by_pattern_batch(hays, overlapping=t == 1) == exp
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ac.count_matches_by_pattern_batch([]) == [0] * len(pats)
