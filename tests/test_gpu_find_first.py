"""GPU tests of find_first (-m gpu): each haystack's first match from acb_find_first + acb_first_rows (the sieve
kernel's first-match mode) and from the table walkers' composition, compared with the CPU oracle's first record per
haystack and with the first row of scan_device, for every match kind.  Also: the skip counters equal what the task
grid predicts, a large haystack stops early, code points, and the window path above one call's range."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, dev, dev_at, forced  # noqa: E402
from .sieve_geometry_helpers import predicted_first_skips  # noqa: E402

ENGINES = ["sieve", "sieve-small-tasks", "staged"]   # the first-match kernel with 16 KiB and 512-byte tasks, the table composition
KIND_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def batch(hays):
    raw = [h.encode() if isinstance(h, str) else bytes(h) for h in hays]
    offs = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=offs[1:])
    data = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)[: offs[-1]].copy()
    return data, offs


def expected(pats, data, offs, kind, codepoints=False):
    """The oracle's first record per haystack, as (n, 3) rows with -1 where there is none."""
    _, counts, rec = Oracle(pats, kind.value).scan_batch(data, offs, codepoints=codepoints)
    rows = np.full((len(offs) - 1, 3), -1, dtype=np.int64)
    at = np.concatenate([[0], np.cumsum(counts.astype(np.int64))[:-1]])
    has = counts > 0
    rows[has] = rec[at[has]][:, 1:4].astype(np.int64)
    return rows


def check(pats, data, offs, kind, shift=None, ac=None):
    """find_first_device equals the oracle's first records and scan_device's first rows.  -> the automaton."""
    exp = expected(pats, data, offs, kind)
    ac = ac or BytesAhoCorasick(pats, kind)
    d = dev_at(data, shift) if shift is not None else dev(data)
    o = dev(offs)
    got = ac.find_first_device(d, o)
    assert got.dtype == torch.int64 and got.shape == (len(offs) - 1, 3)
    got = got.cpu().numpy()
    stats = dict(ac._ac.last_stats)
    assert np.array_equal(got, exp)
    m, mo, total = ac.scan_device(d, o)
    m, mo = m.cpu().numpy().astype(np.int64), mo.cpu().numpy()
    has = mo[1:] > mo[:-1]
    assert np.array_equal(got[has], m[mo[:-1][has]][:, 1:4]) and (got[~has] == -1).all()
    ac._ac.last_stats = stats
    return ac


def engine_of(ac):
    return ac._ac.last_stats["engine"]


# ---------------------------------------------------------------- parity
@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("shortest", range(1, 10))
def test_ragged_small_alphabet(variant, kind, shortest):
    rng = np.random.default_rng(100 + shortest)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 7))).astype(np.uint8)) for _ in range(40)})
    hays = []
    for i in range(300):
        h = rng.integers(97, 101, size=int(rng.integers(0, 40 * shortest + 1))).astype(np.uint8).tobytes() if i % 19 else b""
        if i % 4 == 0 and h:
            at = int(rng.integers(0, len(h) + 1))
            h = h[:at] + pats[i % len(pats)] + h[at:]
        hays.append(h)
    data, offs = batch(hays)
    with forced(variant):
        ac = check(pats, data, offs, kind)
        assert engine_of(ac) == ("table" if variant == "staged" else "sieve")


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_full_byte_range(variant, kind):
    rng = np.random.default_rng(7)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(2, 5))).astype(np.uint8)) for _ in range(300)]
    pats += [b"\x00\xff", b"\xff\x00\x80", b"\x00"]
    data = rng.integers(1, 256, size=400_000, dtype=np.uint8).astype(np.uint8)
    offs = np.unique(np.concatenate([[0, len(data)], rng.integers(0, len(data), size=2000)])).astype(np.int64)
    data[offs[5:40:3]] = 0
    with forced(variant):
        check(pats, data, offs, kind)


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_long_patterns(variant, kind):
    """Patterns of 16 to 1 500 bytes, whole copies and near misses; some of them nested in each other."""
    rng = np.random.default_rng(11)
    pats = [bytes(rng.integers(97, 101, size=int(n)).astype(np.uint8)) for n in (16, 17, 31, 64, 200, 511, 512, 513, 999, 1500)]
    pats += [pats[-1][:700], pats[-1][300:], pats[4][50:150]]
    hays = []
    for i in range(120):
        bg = bytes(rng.integers(97, 101, size=int(rng.integers(0, 3000))).astype(np.uint8))
        p = pats[i % len(pats)]
        piece = p if i % 3 == 0 else (p[:-1] + (b"z" if p[-1:] != b"z" else b"y") if i % 3 == 1 else b"z" + p[1:])
        cut = int(rng.integers(0, len(bg) + 1))
        hays.append(bg[:cut] + piece + bg[cut:])
    data, offs = batch(hays)
    with forced(variant):
        check(pats, data, offs, kind)


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_empty_haystacks(variant, kind):
    pats = [b"abc", b"abcdefgh", b"bcdefghij"]
    hays = [b"", b"ab", b"abc", b"", b"abcdefg", b"bcdefghi", b"xabcx", b"", b"ab" * 2, b"abcdefghij"] + [b""] * 5
    data, offs = batch(hays)
    with forced(variant):
        ac = check(pats, data, offs, kind)
        got = ac.find_first_device(dev(np.zeros(0, dtype=np.uint8)), dev(np.zeros(4, dtype=np.int64)))
        assert got.cpu().tolist() == [[-1, -1, -1]] * 3
        assert ac.find_first_device(dev(data), dev(np.zeros(1, dtype=np.int64))).shape == (0, 3)


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("shift", [0, 1, 255, 511])
def test_matches_straddling_haystacks_do_not_count(variant, kind, shift):
    pats = [b"abcd", b"needle"]
    hays = [b"xxab", b"cdxx", b"xxxnee", b"dlexx", b"a", b"bcd", b"abcd"] * 50
    data, offs = batch(hays)
    with forced(variant):
        ac = check(pats, data, offs, kind, shift=shift)
        got = ac.find_first_device(dev_at(data, shift), dev(offs)).cpu().tolist()
        assert got == ([[-1, -1, -1]] * 6 + [[0, 0, 4]]) * 50


@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("shift", [0, 3, 200, 509])
def test_matches_at_task_grid_edges(variant, kind, shift):
    T = 512 if variant == "sieve-small-tasks" else 16384
    rng = np.random.default_rng(shift)
    pat = b"qrstuvw"
    pats = [pat, b"zz", b"stuv"]
    hays, pos = [], shift
    for i in range(90):
        n = int(rng.integers(20, 2 * T + 600)) if i % 9 else (-pos) % 512 or 512
        h = bytearray(rng.integers(97, 112, size=n).astype(np.uint8).tobytes())
        if i % 3 != 2 and n > 40:
            delta = [-1, 0, 1][i % 3] + ([0, len(pat)][(i // 3) % 2])
            lines = [g for g in range(pos - pos % 512 + 512, pos + n, 512) if pos + 2 <= g - delta and g - delta + len(pat) <= pos + n - 2]
            if lines:
                at = lines[int(rng.integers(0, len(lines)))] - delta - pos
                h[at:at + len(pat)] = pat
        hays.append(bytes(h))
        pos += n
    data, offs = batch(hays)
    with forced(variant):
        assert (expected(pats, data, offs, kind)[:, 0] >= 0).sum() > 30
        ac = check(pats, data, offs, kind, shift=shift)
        assert ac._ac.last_stats["task_bytes"] == T


@pytest.mark.parametrize("variant", ENGINES)
def test_nested_and_duplicate_patterns_differ_by_kind(variant):
    pats = [b"abcd", b"b", b"bcd", b"ab", b"abcd", b"abcdef", b"cdefg"]
    hays = [b"xxabcdefgxx", b"abcd", b"bcdab", b"zzcdefgab", b"q"] * 40
    data, offs = batch(hays)
    with forced(variant):
        answers = [check(pats, data, offs, k).find_first_device(dev(data), dev(offs)).cpu().tolist()[:5] for k in KINDS]
    assert answers[0][0] == [3, 2, 4] and answers[1][0] == [0, 2, 6] and answers[2][0] == [5, 2, 8]
    assert answers[0][1] == [3, 0, 2] and answers[1][1] == [0, 0, 4]   # LeftmostFirst: the lower index of the duplicates
    assert answers[0] != answers[1] != answers[2] != answers[0]


@pytest.mark.parametrize("variant", ["auto", "sieve"])
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_config_shapes_scaled(variant, kind):
    cases = [W.config2(2000), W.config3(n_patterns=2000, n_lines=20_000), W.config5(n_patterns=5000, n_haystacks=2000)]
    for pats, data, offs in cases:
        pats = [p.encode() if isinstance(p, str) else p for p in pats]
        if variant == "auto":
            check(pats, data, offs, kind)
        else:
            with forced("sieve"):
                assert engine_of(check(pats, data, offs, kind)) == "sieve"


# ---------------------------------------------------------------- code points
@pytest.mark.parametrize("variant", ENGINES)
def test_utf8_str_haystacks(variant):
    rng = np.random.default_rng(5)
    alpha = ["a", "b", "é", "—", "☃", "𝄞"]
    pats = sorted({"".join(rng.choice(alpha, size=int(rng.integers(1, 4)))) for _ in range(12)} - {"a", "b"})
    hays = ["".join(rng.choice(alpha, size=int(rng.integers(0, 12)))) for _ in range(400)]
    deep = "ü€" * 220_000 + pats[0] + "é" * 1000   # first match more than 1 MiB in (no pattern uses ü or €)
    hays += [deep, "ü" * 300_000 + pats[-1]]
    with forced(variant):
        for kind in KINDS:
            o = Oracle([p.encode() for p in pats], kind.value)
            exp = [tuple(f[0]) if (f := o.find_str(h)) else None for h in hays]
            assert exp[-2] is not None and len(deep[:exp[-2][1]].encode()) > 1 << 20
            assert 0 < sum(e is not None for e in exp) < len(hays)
            ac = AhoCorasick(pats, kind)
            assert ac.find_first_batch(hays) == exp
            assert [ac.find_first(h) for h in hays[:30] + hays[-2:]] == exp[:30] + exp[-2:]
            data, offs = batch(hays)
            got = ac.find_first_device(dev(data), dev(offs)).cpu().tolist()
            assert got == [list(e) if e else [-1, -1, -1] for e in exp]
            assert got == expected([p.encode() for p in pats], data, offs, kind, codepoints=True).tolist()


# ---------------------------------------------------------------- skip counters and early exit
@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("shift", [0, 188, 511])
def test_entry_keys_skip_exactly(variant, kind, shift):
    """A second call with the first call's keys as entry keys (they cannot be lowered any further) skips exactly what
    the task grid predicts, and returns the same keys."""
    rng = np.random.default_rng(9)
    n, L = 9, 1 << 20
    data = rng.integers(97, 101, size=n * L, dtype=np.uint8).astype(np.uint8)   # a..d: no pattern occurs by chance
    offs = np.arange(n + 1, dtype=np.int64) * L
    pats = [b"abcz", b"zz", b"dcbaz", b"bcz"]
    for h, at in ((0, 100), (2, 300_000), (3, 17_000), (4, L - 10), (6, 600_000), (7, 5)):
        data[h * L + at:h * L + at + 4] = np.frombuffer(b"abcz", dtype=np.uint8)
    data[6 * L + 800_000:6 * L + 800_002] = np.frombuffer(b"zz", dtype=np.uint8)
    ac = BytesAhoCorasick(pats, kind)
    with forced(variant):
        d, o = dev_at(data, shift), dev(offs)
        keys = torch.full((n,), -1, dtype=torch.int64, device="cuda")
        ac._ac.first_keys(d, o, keys)
        rows = ac._ac.first_rows(d, o, keys).cpu().numpy()
        assert np.array_equal(rows, expected(pats, data, offs, kind))
        again = keys.clone()
        scratch = ac._ac.first_keys(d, o, again).cpu().tolist()
        assert torch.equal(again, keys)
        T = ac._ac._plan(d, n).task_bytes
        assert T == (512 if variant == "sieve-small-tasks" else 16384)
        key_hi = keys.cpu().numpy().view(np.uint64) >> np.uint64(32)
        tasks, windows = predicted_first_skips(d.data_ptr(), offs, key_hi, T, kind, ac._ac.max_pattern_len)
        assert (scratch[1], scratch[2]) == (tasks, windows)
        assert tasks > 0
        if shift and T > 512:
            assert windows > 0


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_one_large_haystack_stops_early(kind):
    n = 256 << 20   # (far more tasks than the grid has warps: most are claimed after the key is set)
    ac = BytesAhoCorasick([b"needle", b"haystack", b"needle in"], kind)
    offs = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    hay = torch.full((n,), ord("x"), dtype=torch.uint8, device="cuda")
    put = lambda at, b: hay[at:at + len(b)].copy_(torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda())  # noqa: E731
    with forced("sieve"):
        assert ac.find_first_device(hay, offs).cpu().tolist() == [[-1, -1, -1]]
        skipped = ac._ac.last_stats["skip_counters"].cpu().tolist()
        assert skipped[1] == 0 and skipped[2] == 0
        put(700, b"needle in")
        put(5000, b"haystack")
        want = {MatchKind.Standard: [0, 700, 706], MatchKind.LeftmostFirst: [0, 700, 706], MatchKind.LeftmostLongest: [2, 700, 709]}[kind]
        assert ac.find_first_device(hay, offs).cpu().tolist() == [want]
        st = ac._ac.last_stats
        assert st["skip_counters"].cpu().tolist()[1] > st["tasks"] // 2, st
        hay[700:709] = ord("x")
        hay[5000:5008] = ord("x")
        put(n - 8, b"haystack")
        assert ac.find_first_device(hay, offs).cpu().tolist() == [[1, n - 8, n]]
    del hay


# ---------------------------------------------------------------- windows and runs above one call's range
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_windows_and_runs_match_one_call(kind, monkeypatch):
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    data, offs = W.ragged(400, 3000, b"abcdxyz", seed=32)
    ac = BytesAhoCorasick(pats, kind)
    one = ac.find_first_device(dev(data), dev(offs)).cpu().numpy()
    assert np.array_equal(one, expected(pats, data, offs, kind)) and (one[:, 0] >= 0).any() and (one[:, 0] < 0).any()
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
    assert np.array_equal(ac.find_first_device(dev(data), dev(offs)).cpu().numpy(), one)


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_oversized_haystack_in_windows(kind, monkeypatch):
    """One haystack above the window limit among small ones.  Window 0 sees only the short pattern at p (the long one
    runs past its end); p lies in the bytes window 0 shares with window 1, which sees both: the leftmost kinds must
    look at window 1 and pick the long one there, Standard stops at window 0."""
    limit = 30_001
    long_, short = b"needle12345", b"needle"
    pats = [long_, short] if kind == MatchKind.LeftmostFirst else [short, long_]
    halo = len(long_) - 1
    step = limit - halo
    p = limit - 8
    assert step <= p and p + len(short) <= limit < p + len(long_)
    big = bytearray(b"x" * 200_000)
    big[p:p + len(long_)] = long_
    big[150_000:150_000 + len(long_)] = long_
    hays = [b"xneedle", b"xx", bytes(big), b"needle1", b"yy" * 3, bytes(b"z" * 70_000) + long_]
    data, offs = batch(hays)
    exp = expected(pats, data, offs, kind)
    # LeftmostFirst: the long pattern has the lower index; LeftmostLongest: it is longer; Standard: the short one ends first
    assert exp[2].tolist() == ([0, p, p + 6] if kind == MatchKind.Standard else
                               [0, p, p + 11] if kind == MatchKind.LeftmostFirst else [1, p, p + 11])
    ac = BytesAhoCorasick(pats, kind)
    assert np.array_equal(ac.find_first_device(dev(data), dev(offs)).cpu().numpy(), exp)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", limit)
    for variant in ("sieve", "staged"):
        with forced(variant):
            assert np.array_equal(ac.find_first_device(dev(data), dev(offs)).cpu().numpy(), exp)
            assert ac.find_first(bytes(big)) == tuple(exp[2].tolist())
            n0 = _capi.lib().acb_launch_count()
            assert ac.find_first(b"x" * 100_000) is None
            assert _capi.lib().acb_launch_count() > n0


def test_oversized_utf8_haystack_in_windows(monkeypatch):
    """Code points are converted once, over the whole buffer, with 64-bit positions."""
    pats = ["☃x", "needle"]
    hay = "é" * 40_000 + "☃" * 10 + "needle" + "é" * 5000
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 30_001)
    for kind in KINDS:
        want = tuple(Oracle([p.encode() for p in pats], kind.value).find_str(hay)[0])
        assert AhoCorasick(pats, kind).find_first(hay) == want == (1, 40_010, 40_016)


# ---------------------------------------------------------------- engine selection, launches, threads
def test_engine_follows_the_scan_rule(monkeypatch):
    pats, data, offs = W.config2(1100)
    pats = [p.encode() for p in pats]
    assert data.nbytes >= matcher._Automaton.AUTO_PROFILE_BYTES
    for kind in KINDS:
        ac = BytesAhoCorasick(pats, kind)
        check(pats, data, offs, kind, ac=ac)
        assert engine_of(ac) == "table" and ac._ac.last_stats["mode"] == "first"
    monkeypatch.setattr(matcher._Automaton, "ENGINE", "sieve")
    got = ac.find_first_device(dev(data), dev(offs))
    assert engine_of(ac) == "sieve" and np.array_equal(got.cpu().numpy(), expected(pats, data, offs, kind))


def test_launches_per_sieve_call():
    pats, data, offs = W.config3(n_patterns=500, n_lines=2000)
    d, o = dev(data), dev(offs)
    L = _capi.lib()
    with forced("sieve"):
        for kind in KINDS:
            ac = BytesAhoCorasick(pats, kind)
            exp = expected(pats, data, offs, kind)
            ac.find_first_device(d, o)
            n0 = L.acb_launch_count()
            for _ in range(3):
                got = ac.find_first_device(d, o)
            assert L.acb_launch_count() == n0 + 6   # acb_find_first + acb_first_rows
            assert np.array_equal(got.cpu().numpy(), exp)
            sac = AhoCorasick([p.decode() for p in pats], kind)
            sac.find_first_device(d, o)
            n0 = L.acb_launch_count()
            sac.find_first_device(d, o)
            assert L.acb_launch_count() == n0 + 3   # ... + acb_rows_to_codepoints


def test_two_threads_share_one_automaton():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(3, 7))).astype(np.uint8)) for _ in range(60)})
    ac = BytesAhoCorasick(pats, MatchKind.LeftmostLongest)
    inputs = []
    for t in range(2):
        data, offs = W.ragged(300, 200 + 100 * t, b"abcdxyz", seed=50 + t)
        hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
        exp = [tuple(r) if r[0] >= 0 else None for r in expected(pats, data, offs, MatchKind.LeftmostLongest).tolist()]
        inputs.append((hays, exp))
    errors = []

    def work(t):
        try:
            hays, exp = inputs[t]
            for _ in range(25):
                assert ac.find_first_batch(hays) == exp
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ac.find_first_batch([]) == []
