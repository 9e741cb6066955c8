"""GPU tests of matching_patterns (-m gpu): each haystack's distinct patterns with their counts, from acb_pattern_hits
(the sieve's list scan and the hits epilogue: warp-sorted short stretches, counter rows for long ones) and the table
walkers' composition.  The expected answer is always Counter of the oracle's pattern column per haystack.  Also: the
row and column sums against count_matches_device and count_matches_by_pattern_device, the sparse CSR matrix,
stretches around ACB_LONG_STRETCH records, 400 k-record haystacks next to short ones, a hot pattern, retries for a
small workspace and small counter rows, runs and windows above one call's range, the golden vectors and two threads."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, SEARCH_IDS, SEARCHES, dev, forced  # noqa: E402
from .sieve_geometry_helpers import oracle_hits  # noqa: E402
from .test_gpu_count import ENGINES, KIND_IDS, L_STRETCH, VECTORS, batch, stretch_batch  # noqa: E402


def check(pats, data, offs, kind, overlapping=False, ac=None, capacity=None, sums=True):
    """matching_patterns_device equals the oracle's hits; its row sums equal count_matches_device and its column sums
    count_matches_by_pattern_device.  -> (ac, last_stats)."""
    exp = oracle_hits(pats, data, offs, kind, overlapping)
    ac = ac or BytesAhoCorasick(pats, kind)
    d, o = dev(data), dev(offs)
    got = ac.matching_patterns_device(d, o, overlapping) if capacity is None else ac._ac.hits_device(d, o, overlapping, capacity)
    stats = dict(ac._ac.last_stats)
    assert stats["mode"] == "matching_patterns"
    n, k = len(offs) - 1, len(exp[1])
    for t, shape, want in zip(got, [(n + 1,), (k,), (k,)], exp):
        assert t.dtype == torch.int64 and t.shape == shape and t.device == d.device
        assert np.array_equal(t.cpu().numpy(), want)
    assert stats["hits"] == k
    if sums:
        ro, p, c = got
        rows = torch.zeros(n, dtype=torch.int64, device=d.device).index_add_(0, torch.repeat_interleave(
            torch.arange(n, device=d.device), ro[1:] - ro[:-1]), c)
        assert torch.equal(rows, ac.count_matches_device(d, o, overlapping))
        cols = torch.zeros(len(pats), dtype=torch.int64, device=d.device).index_add_(0, p, c)
        assert torch.equal(cols, ac.count_matches_by_pattern_device(d, o, overlapping))
    return ac, stats


# ---------------------------------------------------------------- parity
@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("shortest", [1, 2, 3, 5])
def test_ragged_small_alphabet(variant, search, shortest):
    kind, overlapping = search
    rng = np.random.default_rng(600 + shortest)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 7))).astype(np.uint8)) for _ in range(40)})
    pats += pats[:2]   # duplicates: distinct ids, same bytes
    hays = []
    for i in range(300):
        h = rng.integers(97, 101, size=int(rng.integers(0, 60 * shortest + 1))).astype(np.uint8).tobytes() if i % 19 else b""
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
def test_full_byte_range_and_empty_haystacks(variant, search):
    kind, overlapping = search
    rng = np.random.default_rng(17)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(2, 5))).astype(np.uint8)) for _ in range(300)]
    pats += [b"\x00\xff", b"\xff\x00\x80", b"\x00", b"abcd", b"\x00"]
    data = rng.integers(1, 256, size=300_000, dtype=np.uint8).astype(np.uint8)
    offs = np.unique(np.concatenate([[0, len(data)], rng.integers(0, len(data), size=2000)])).astype(np.int64)
    offs = np.sort(np.concatenate([offs, offs[10:200:7]]))   # empty haystacks
    data[offs[5:40:3]] = 0
    with forced(variant):
        check(pats, data, offs, kind, overlapping)
        d2, o2 = batch([b"xxab", b"cdxx", b"a", b"bcd", b"abcd", b""] * 40)   # matches across haystacks never count
        check(pats, d2, o2, kind, overlapping)


def test_sort_paths_of_short_stretches():
    """Selections of 1..32 pids (registers), 33..1024 (the warp's shared buffer) and 1025..4096 (the stretch's slice
    of raw_seq), with many distinct patterns and repeats, on the sieve."""
    pats = [bytes([97 + i // 26, 97 + i % 26]) for i in range(26 * 26)] + [b"a", b"zz", b"aa"]
    rng = np.random.default_rng(3)
    hays = []
    for size in (1, 2, 16, 40, 300, 700, 1100, 1500, 1900):
        hays.append(bytes(rng.integers(97, 123, size=size).astype(np.uint8)))
        hays.append(b"")
    data, offs = batch(hays)
    with forced("sieve"):
        for kind, overlapping in SEARCHES:
            _, st = check(pats, data, offs, kind, overlapping)
            assert st["long_stretches"] == 0 and st["rows"] == 0


# ---------------------------------------------------------------- counter rows for long stretches
@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_stretches_around_the_long_stretch_limit(variant, search):
    kind, overlapping = search
    rng = np.random.default_rng(5)
    hays, n_long = stretch_batch(rng)
    pats = [b"a", b"aa", b"b"] if kind != MatchKind.LeftmostFirst else [b"aa", b"a", b"b"]
    data, offs = batch(hays)
    with forced(variant):
        ac, st = check(pats, data, offs, kind, overlapping)
        assert st["long_stretches"] == n_long and st["rows"] == n_long, st
        for h, want in ((b"a" * (L_STRETCH // 2), 0), (b"a" * (L_STRETCH // 2) + b"b", 0), (b"a" * (L_STRETCH // 2 + 1), 1)):
            d, o = batch([h])
            _, st = check(pats, d, o, kind, overlapping, ac=ac)
            assert st["long_stretches"] == want and st["rows"] == want


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_dense_haystacks_next_to_short_ones(search):
    """400 k-record haystacks with nested and self-overlapping patterns (and a duplicate) next to short haystacks, and
    a pattern set of 3 000 (rows of two counter tiles)."""
    kind, overlapping = search
    rng = np.random.default_rng(9)
    pats = [b"ab", b"aba", b"bab", b"abab", b"b", b"baab", b"aa", b"ab"]
    pats += [bytes(rng.integers(99, 123, size=6).astype(np.uint8)) for _ in range(3000)] + [b"ba"]
    big = rng.choice(list(b"ab"), size=400_000).astype(np.uint8).tobytes()
    hays = [b"abab", big, b"", b"babab" * 10, big[:70_000] + pats[20] + pats[3000], b"x"]
    data, offs = batch(hays)
    with forced("sieve"):
        _, st = check(pats, data, offs, kind, overlapping)
        assert st["long_stretches"] == 2 and st["rows"] == 2 and st["list_records"] > 300_000


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_hot_pattern(search):
    """One single-byte pattern (twice: two ids) matching every position of 24 MiB plus a few rare ones."""
    kind, overlapping = search
    data = np.full(24 << 20, ord("a"), dtype=np.uint8)
    rng = np.random.default_rng(12)
    pos = np.sort(rng.choice(len(data) // 8, size=300, replace=False)) * 8
    for k, p in enumerate(pos):
        data[p:p + 5] = np.frombuffer([b"xqzjk", b"vwxyz"][k % 2], dtype=np.uint8)
    pats = [b"a", b"xqzjk", b"vwxyz", b"zzqzz", b"a"]
    offs = np.array([0, 1 << 20, 13 << 20, 13 << 20, len(data) - 3, len(data)], dtype=np.int64)
    with forced("sieve"):
        _, st = check(pats, data, offs, kind, overlapping)
        assert st["rows"] == 3


def test_sparse_csr_matrix():
    pats = [b"ab", b"b", b"ab", b"xyz", b"a"]
    hays = [b"abab", b"", b"xyzb", b"zzz", b"aab" * 3]
    data, offs = batch(hays)
    for kind, overlapping in SEARCHES:
        ac = BytesAhoCorasick(pats, kind)
        ro, p, c = ac.matching_patterns_device(dev(data), dev(offs), overlapping)
        m = torch.sparse_csr_tensor(ro, p, c, size=(len(hays), len(pats)))
        want = np.zeros((len(hays), len(pats)), dtype=np.int64)
        for h, hay in enumerate(hays):
            for pid, _, _ in Oracle(pats, kind.value).find(hay, overlapping=overlapping):
                want[h, pid] += 1
        assert np.array_equal(m.to_dense().cpu().numpy(), want)
        assert np.array_equal(torch.bincount(p, minlength=len(pats)).cpu().numpy(), (want > 0).sum(axis=0))


# ---------------------------------------------------------------- retries
def test_small_workspace_and_small_rows_retry_to_the_same_answer():
    pats = [b"a", b"aa", b"b", b"ab"]
    data, offs = batch([b"a" * 30_000, b"ab" * 100, b"b" * 5000, b"", b"a" * 9000 + b"b"])
    L = _capi.lib()
    with forced("sieve"):
        for kind, overlapping in SEARCHES:
            ac = BytesAhoCorasick(pats, kind)
            n0 = L.acb_launch_count()
            _, st = check(pats, data, offs, kind, overlapping, ac=ac, capacity=1)   # no rows yet, a list that does not fit
            assert L.acb_launch_count() >= n0 + 6 and st["rows"] >= 2
    # direct calls: a list that does not fit, then rows one word short; nothing valid is reported until both fit
    ac = BytesAhoCorasick(pats, MatchKind.LeftmostLongest)
    a = ac._ac
    d, o = dev(data), dev(offs)
    n = len(offs) - 1
    with forced("sieve"), torch.cuda.device(d.device):
        sieve_t, _ = a.sieve(d.device)
        plan = a._plan(d, n)
        stream = torch.cuda.current_stream(d.device).cuda_stream

        def call(cap, words):
            ws = a._workspace(d.device, plan, n, cap, 0)
            st = a._ws_struct(ws)
            rows = torch.empty(max(words, 2), dtype=torch.int32, device=d.device)
            assert a._L.acb_pattern_hits(a._h, sieve_t.data_ptr(), d.data_ptr(), o.data_ptr(), n, d.numel(), 0, C.byref(plan),
                                         C.byref(st), rows.data_ptr(), words, stream) == _capi.ACB_OK, _capi.last_error()
            return ws, ws["total"].tolist()

        _, tot = call(16, 0)
        assert tot[1] == 0 and tot[0] == 0 and tot[4] > 16
        room = tot[4]
        _, tot = call(room, 0)
        assert tot[1] == 0 and tot[2] == 3 and tot[3] == 0
        need = tot[5]
        assert need == 3 * (4 + 2 + 2)   # acb_pattern_hit_row_words(4) per long stretch
        _, tot = call(room, need - 1)
        assert tot[1] == 0 and tot[5] == need
        ws, tot = call(room, need)
        assert tot[1] == 1 and tot[2] == tot[3] == 3
        exp = oracle_hits(pats, data, offs, MatchKind.LeftmostLongest, False)
        k = tot[0]
        assert k == len(exp[1])
        out = ws["out"][:k].cpu().numpy()
        assert np.array_equal(out[:, 1], exp[1]) and np.array_equal(out[:, 2], exp[2]) and not out[:, 3].any()
        assert np.array_equal(ws["match_offsets"][: n + 1].cpu().numpy(), exp[0])


# ---------------------------------------------------------------- runs and windows above one call's range
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_windows_and_runs(search, monkeypatch):
    kind, overlapping = search
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    data, offs = W.ragged(400, 3000, b"abcdxyz", seed=32)
    exp = oracle_hits(pats, data, offs, kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
    got = ac.matching_patterns_device(dev(data), dev(offs), overlapping)
    assert ac._ac.last_stats["windows"]
    for t, want in zip(got, exp):
        assert np.array_equal(t.cpu().numpy(), want)


@pytest.mark.parametrize("variant", ["sieve", "staged"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_oversized_haystack_in_windows(variant, search, monkeypatch):
    """One haystack above the window limit among small ones, with matches inside the bytes windows share."""
    kind, overlapping = search
    limit = 30_001
    pats = [b"needle12345", b"needle", b"aa", b"a", b"needle", b"zzz"]
    rng = np.random.default_rng(8)
    big = bytearray(rng.choice(list(b"xa"), size=200_000).astype(np.uint8).tobytes())
    step = limit - (len(pats[0]) - 1)
    for p in (limit - 8, step - 3, 2 * step + 1, 150_000):
        big[p:p + 11] = pats[0]
    hays = [b"xneedle", b"xx", bytes(big), b"needle1", b"aaaa", bytes(b"a" * 70_000) + pats[0], b""]
    data, offs = batch(hays)
    exp = oracle_hits(pats, data, offs, kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", limit)
    with forced(variant):
        got = ac.matching_patterns_device(dev(data), dev(offs), overlapping)
        for t, want in zip(got, exp):
            assert np.array_equal(t.cpu().numpy(), want)
        assert ac.matching_patterns(bytes(big), overlapping) == exp[1][exp[0][2]:exp[0][3]].tolist()


# ---------------------------------------------------------------- code points, golden vectors
def test_utf8_haystacks_on_the_str_class():
    pats = ["é", "éé", "☃x", "needle", "x", "é"]
    hays = ["", "é" * 500, "☃x" * 40 + "needle", "aé☃xé" * 300, "x" * 10_000, "ascii only"]
    for variant in ENGINES:
        with forced(variant):
            for kind in KINDS:
                ac = AhoCorasick(pats, kind)
                for overlapping in ([False, True] if kind == MatchKind.Standard else [False]):
                    want = [sorted({m[0] for m in ac.find_matches_as_indexes(h, overlapping)}) for h in hays]
                    assert ac.matching_patterns_batch(hays, overlapping) == want
                    assert ac.matching_patterns(hays[3], overlapping) == want[3]
                    data, offs = batch(hays)
                    ro, p, _ = ac.matching_patterns_device(dev(data), dev(offs), overlapping)
                    ro, p = ro.cpu().tolist(), p.cpu().tolist()
                    assert [p[ro[h]:ro[h + 1]] for h in range(len(hays))] == want


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
                    ac.matching_patterns(hay, overlapping=True)
                continue
            want = sorted({m[0] for m in ac.find_matches_as_indexes(hay, overlapping=vec["overlapping"])})
            if "expect_indexes" in vec:
                assert want == sorted({m[0] for m in vec["expect_indexes"]})
            assert ac.matching_patterns(hay, overlapping=vec["overlapping"]) == want, vec
            assert ac.matching_patterns_batch([hay, hay], overlapping=vec["overlapping"]) == [want, want]


# ---------------------------------------------------------------- threads
def test_two_threads_share_one_automaton():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(2, 7))).astype(np.uint8)) for _ in range(60)})
    ac = BytesAhoCorasick(pats, MatchKind.Standard)
    inputs = []
    for t in range(2):
        data, offs = W.ragged(300, 200 + 100 * t, b"abcdxyz", seed=50 + t)
        hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
        ro, p, _ = oracle_hits(pats, data, offs, MatchKind.Standard, t == 1)
        inputs.append((hays, [p[ro[h]:ro[h + 1]].tolist() for h in range(len(hays))]))
    errors = []

    def work(t):
        try:
            hays, exp = inputs[t]
            for _ in range(25):
                assert ac.matching_patterns_batch(hays, overlapping=t == 1) == exp
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ac.matching_patterns_batch([]) == []
