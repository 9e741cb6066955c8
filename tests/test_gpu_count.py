"""GPU tests of count_matches (-m gpu): per-haystack match counts from acb_count_overlapping (the sieve kernel's count
mode), acb_count_non_overlapping (the sieve's list scan and the count epilogue, serial and grid-wide stretches) and
the table walkers' composition, compared with the CPU oracle's counts and with diff(match_offsets) of scan_device, for
every match kind and both searches.  Also: stretches around ACB_LONG_STRETCH records, a workspace retry, code points,
the golden vectors, the window path above one call's range, config 4 at size and two threads."""
import json
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, Implementation, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, SEARCH_IDS, SEARCHES, dev, forced  # noqa: E402

ENGINES = ["sieve", "sieve-small-tasks", "staged"]   # the count kernels with 16 KiB and 512-byte tasks, the table composition
KIND_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]
L_STRETCH = _capi.ACB_LONG_STRETCH
HERE = os.path.dirname(os.path.abspath(__file__))


def batch(hays):
    raw = [h.encode() if isinstance(h, str) else bytes(h) for h in hays]
    offs = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=offs[1:])
    data = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)[: offs[-1]].copy()
    return data, offs


def oracle_counts(pats, data, offs, kind, overlapping):
    _, counts, _ = Oracle(pats, kind.value).scan_batch(data, offs, overlapping=overlapping, want_records=False)
    return counts.astype(np.int64)


def check(pats, data, offs, kind, overlapping=False, ac=None, capacity=None):
    """count_matches_device equals the oracle's counts and diff(match_offsets) of scan_device.  -> (ac, last_stats)."""
    exp = oracle_counts(pats, data, offs, kind, overlapping)
    ac = ac or BytesAhoCorasick(pats, kind)
    d, o = dev(data), dev(offs)
    got = ac.count_matches_device(d, o, overlapping) if capacity is None else ac._ac.count_device(d, o, overlapping, capacity)
    assert got.dtype == torch.int64 and got.shape == (len(offs) - 1,)
    got = got.cpu().numpy()
    stats = dict(ac._ac.last_stats)
    assert stats["mode"] == "count"
    assert np.array_equal(got, exp)
    _, mo, _ = ac.scan_device(d, o, overlapping)
    assert np.array_equal(np.diff(mo.cpu().numpy()), got)
    return ac, stats


# ---------------------------------------------------------------- parity
@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("shortest", range(1, 10))
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
    pats += [b"\x00\xff", b"\xff\x00\x80", b"\x00", b"abcd"]
    data = rng.integers(1, 256, size=300_000, dtype=np.uint8).astype(np.uint8)
    offs = np.unique(np.concatenate([[0, len(data)], rng.integers(0, len(data), size=2000)])).astype(np.int64)
    data[offs[5:40:3]] = 0
    with forced(variant):
        check(pats, data, offs, kind, overlapping)
        d2, o2 = batch([b"xxab", b"cdxx", b"a", b"bcd", b"abcd", b""] * 40)   # matches across haystacks never count
        check(pats, d2, o2, kind, overlapping)


# ---------------------------------------------------------------- the parallel path for long stretches
def stretch_batch(rng):
    """Haystacks whose overlapping lists (patterns a, aa, b) hold L - 1, L and L + 1 records, a few hundred thousand,
    and short ones in between.  "a" * m has 2 m - 1 records; a trailing b adds one."""
    m = L_STRETCH // 2
    long_hays = [b"a" * m, b"a" * m + b"b", b"a" * (m + 1), b"ab" * 3 + b"a" * 150_000 + b"b"]
    sizes = [2 * m - 1, 2 * m, 2 * m + 1]
    assert sizes == [L_STRETCH - 1, L_STRETCH, L_STRETCH + 1]
    hays = []
    for h in long_hays:
        hays += [bytes(rng.choice(list(b"abx"), size=int(rng.integers(0, 50))).astype(np.uint8)) for _ in range(30)]
        hays.append(h)
    return hays, 2   # L + 1 and the last one are counted by the grid


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
        # each long haystack alone: its stretch reaches the path it targets
        for h, want in ((b"a" * (L_STRETCH // 2), 0), (b"a" * (L_STRETCH // 2) + b"b", 0), (b"a" * (L_STRETCH // 2 + 1), 1)):
            d, o = batch([h])
            check(pats, d, o, kind, ac=ac)
            ac.count_matches_device(dev(d), dev(o))
            assert ac._ac.last_stats["long_stretches"] == want


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_dense_single_haystacks_on_the_grid(kind):
    """Hundreds of thousands of records in one haystack, with nested and self-overlapping patterns: the leftmost kinds'
    look-ahead and restarts inside the list, next to short haystacks in the same batch."""
    rng = np.random.default_rng(9)
    pats = [b"ab", b"aba", b"bab", b"abab", b"b", b"baab", b"aa", b"ab"]
    big = rng.choice(list(b"ab"), size=400_000).astype(np.uint8).tobytes()
    hays = [b"abab", big, b"", b"babab" * 10, big[:70_000], b"x"]
    data, offs = batch(hays)
    with forced("sieve"):
        _, st = check(pats, data, offs, kind)
        assert st["long_stretches"] == 2 and st["list_records"] > 300_000


def test_workspace_retry():
    pats = [b"a", b"aa", b"b"]
    data, offs = batch([b"a" * 30_000, b"ab" * 100, b"b" * 5000])
    L = _capi.lib()
    with forced("sieve"):
        for kind in KINDS:
            ac = BytesAhoCorasick(pats, kind)
            n0 = L.acb_launch_count()
            check(pats, data, offs, kind, ac=ac, capacity=1)
            assert L.acb_launch_count() >= n0 + 4   # (the list did not fit: scan + epilogue twice)
            n0 = L.acb_launch_count()
            ac.count_matches_device(dev(data), dev(offs))
            assert L.acb_launch_count() == n0 + 2   # the workspace has grown: one scan + one epilogue
            ac.count_matches_device(dev(data), dev(offs), overlapping=kind == MatchKind.Standard)
            if kind == MatchKind.Standard:
                assert L.acb_launch_count() == n0 + 3   # the count mode: one launch


# ---------------------------------------------------------------- code points, golden vectors
def test_utf8_haystacks_on_the_str_class():
    pats = ["é", "éé", "☃x", "needle", "x"]
    hays = ["", "é" * 500, "☃x" * 40 + "needle", "aé☃xé" * 300, "x" * 10_000, "ascii only"]
    for variant in ENGINES:
        with forced(variant):
            for kind in KINDS:
                ac = AhoCorasick(pats, kind)
                searches = [False, True] if kind == MatchKind.Standard else [False]
                for overlapping in searches:
                    want = [len(ac.find_matches_as_indexes(h, overlapping)) for h in hays]
                    assert ac.count_matches_batch(hays, overlapping) == want
                    assert [ac.count_matches(h, overlapping) for h in hays] == want
                    data, offs = batch(hays)
                    assert ac.count_matches_device(dev(data), dev(offs), overlapping).cpu().tolist() == want


with open(os.path.join(HERE, "golden", "reference_vectors.json"), encoding="utf-8") as f:
    VECTORS = json.load(f)["vectors"]


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
                    ac.count_matches(hay, overlapping=True)
                continue
            want = len(ac.find_matches_as_indexes(hay, overlapping=vec["overlapping"]))
            if "expect_indexes" in vec:
                assert want == len(vec["expect_indexes"])
            assert ac.count_matches(hay, overlapping=vec["overlapping"]) == want, vec


# ---------------------------------------------------------------- windows and runs above one call's range
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_windows_and_runs(search, monkeypatch):
    kind, overlapping = search
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    data, offs = W.ragged(400, 3000, b"abcdxyz", seed=32)
    exp = oracle_counts(pats, data, offs, kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    assert np.array_equal(ac.count_matches_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
    assert np.array_equal(ac.count_matches_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
    assert ac._ac.last_stats["windows"]


@pytest.mark.parametrize("variant", ["sieve", "staged"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_oversized_haystack_in_windows(variant, search, monkeypatch):
    """One haystack above the window limit among small ones, with matches inside the bytes windows share (counted
    once) and a dense stretch; the non-overlapping count goes through acb_count_rows."""
    kind, overlapping = search
    limit = 30_001
    pats = [b"needle12345", b"needle", b"aa", b"a"]
    rng = np.random.default_rng(8)
    big = bytearray(rng.choice(list(b"xa"), size=200_000).astype(np.uint8).tobytes())
    step = limit - (len(pats[0]) - 1)
    for p in (limit - 8, step - 3, 2 * step + 1, 150_000):
        big[p:p + 11] = pats[0]
    hays = [b"xneedle", b"xx", bytes(big), b"needle1", b"aaaa", bytes(b"a" * 70_000) + pats[0]]
    data, offs = batch(hays)
    exp = oracle_counts(pats, data, offs, kind, overlapping)
    ac = BytesAhoCorasick(pats, kind)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", limit)
    with forced(variant):
        assert np.array_equal(ac.count_matches_device(dev(data), dev(offs), overlapping).cpu().numpy(), exp)
        assert ac.count_matches(bytes(big), overlapping) == exp[2]
        _, mo, _ = ac.scan_device(dev(data), dev(offs), overlapping)
        assert np.array_equal(np.diff(mo.cpu().numpy()), exp)


def test_config4_single_4gib_haystack_overlapping():
    """BASELINE config 4 at size: ONE haystack of 2^32 bytes, 100k patterns, overlapping, counted in windows; equal to
    the total of scan_device's list."""
    n = 1 << 32
    pats = W.random_lowercase_patterns(100_000, 5, 8, 4)
    g = torch.Generator(device="cuda")
    g.manual_seed(1004)
    d = torch.empty(n, dtype=torch.uint8, device="cuda")
    for a in range(0, n, 1 << 28):
        d[a:a + (1 << 28)] = torch.randint(97, 123, (1 << 28,), dtype=torch.uint8, device="cuda", generator=g)
    ac = BytesAhoCorasick(pats, implementation=Implementation.ContiguousNFA)
    o = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    got = ac.count_matches_device(d, o, overlapping=True).cpu().tolist()
    _, mo, total = ac.scan_device(d, o, overlapping=True)
    assert got == [total] and total > 5_000_000
    del d


# ---------------------------------------------------------------- threads
def test_two_threads_share_one_automaton():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(2, 7))).astype(np.uint8)) for _ in range(60)})
    ac = BytesAhoCorasick(pats, MatchKind.Standard)
    inputs = []
    for t in range(2):
        data, offs = W.ragged(300, 200 + 100 * t, b"abcdxyz", seed=50 + t)
        hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
        inputs.append((hays, oracle_counts(pats, data, offs, MatchKind.Standard, t == 1).tolist()))
    errors = []

    def work(t):
        try:
            hays, exp = inputs[t]
            for _ in range(25):
                assert ac.count_matches_batch(hays, overlapping=t == 1) == exp
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ac.count_matches_batch([]) == []
