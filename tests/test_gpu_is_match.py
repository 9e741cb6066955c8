"""GPU tests of is_match (-m gpu): the per-haystack "contains any pattern" flags of acb_any_match (the sieve kernel's
any-match mode) and of the table walkers' composition, compared with the CPU oracle's per-haystack counts and, for
small inputs, with `any(p in hay for p in patterns)`.  Also: the flags do not depend on the match kind, the skip
counters equal what the task grid predicts, a large haystack stops early, and the window path above one call's
range gives what one call gives."""
import contextlib
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import KINDS, dev, dev_at, forced  # noqa: E402
from .sieve_geometry_helpers import predicted_any_skips  # noqa: E402

ENGINES = ["sieve", "sieve-small-tasks", "staged"]   # the any-match kernel with 16 KiB and 512-byte tasks, the table composition
SPEC_BYTES = 8192


def batch(hays):
    raw = [h.encode() if isinstance(h, str) else bytes(h) for h in hays]
    offs = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=offs[1:])
    data = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)[: offs[-1]].copy()
    return data, offs


def expected(pats, data, offs):
    _, counts, _ = Oracle(pats, "Standard").scan_batch(data, offs, want_records=False)
    exp = counts > 0
    if int(offs[-1] - offs[0]) <= SPEC_BYTES:
        brute = [any(p in data[offs[h]:offs[h + 1]].tobytes() for p in pats) for h in range(len(offs) - 1)]
        assert exp.tolist() == brute
    return exp


def check(pats, data, offs, shift=None, kind=MatchKind.Standard, ac=None):
    """is_match_device on (data, offs) equals the oracle's counts > 0.  -> the automaton (last_stats describe the call)."""
    exp = expected(pats, data, offs)
    ac = ac or BytesAhoCorasick(pats, kind)
    d = dev_at(data, shift) if shift is not None else dev(data)
    got = ac.is_match_device(d, dev(offs))
    assert got.dtype == torch.bool and got.shape == (len(offs) - 1,)
    assert np.array_equal(got.cpu().numpy(), exp)
    return ac


def engine_of(ac):
    return ac._ac.last_stats["engine"]


# ---------------------------------------------------------------- parity
@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("shortest", range(1, 10))
def test_ragged_small_alphabet(variant, shortest):
    rng = np.random.default_rng(100 + shortest)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 7))).astype(np.uint8)) for _ in range(40)})
    hays = []
    for i in range(300):
        h = rng.integers(97, 101, size=int(rng.integers(0, 40 * shortest + 1))).astype(np.uint8).tobytes() if i % 19 else b""
        if i % 4 == 0 and h:   # plant a pattern: long shortest patterns seldom occur by chance
            at = int(rng.integers(0, len(h) + 1))
            h = h[:at] + pats[i % len(pats)] + h[at:]
        hays.append(h)
    data, offs = batch(hays)
    with forced(variant):
        exp = expected(pats, data, offs)
        assert 0 < exp.sum() < len(exp)
        ac = check(pats, data, offs)
        assert engine_of(ac) == ("table" if variant == "staged" else "sieve")
        small = data[: offs[20]], offs[:21]
        check(pats, *small, ac=ac)


@pytest.mark.parametrize("variant", ENGINES)
def test_full_byte_range(variant):
    rng = np.random.default_rng(7)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(2, 5))).astype(np.uint8)) for _ in range(300)]
    pats += [b"\x00\xff", b"\xff\x00\x80", b"\x00"]
    data = rng.integers(1, 256, size=400_000, dtype=np.uint8).astype(np.uint8)
    offs = np.unique(np.concatenate([[0, len(data)], rng.integers(0, len(data), size=2000)])).astype(np.int64)
    data[offs[5:40:3]] = 0   # a few NUL bytes for the one-byte pattern
    with forced(variant):
        check(pats, data, offs)


@pytest.mark.parametrize("variant", ENGINES)
def test_long_patterns(variant):
    """Patterns of 16 to 1 500 bytes (longer than the sieve's on-chip levels), whole copies and near misses."""
    rng = np.random.default_rng(11)
    pats = [bytes(rng.integers(97, 101, size=int(n)).astype(np.uint8)) for n in (16, 17, 31, 64, 200, 511, 512, 513, 999, 1500)]
    hays = []
    for i in range(120):
        bg = bytes(rng.integers(97, 101, size=int(rng.integers(0, 3000))).astype(np.uint8))
        p = pats[i % len(pats)]
        if i % 3 == 0:
            piece = p
        elif i % 3 == 1:
            piece = p[:-1] + (b"z" if p[-1:] != b"z" else b"y")   # last byte wrong
        else:
            piece = b"z" + p[1:]                                  # first byte wrong
        cut = int(rng.integers(0, len(bg) + 1))
        hays.append(bg[:cut] + piece + bg[cut:])
    data, offs = batch(hays)
    with forced(variant):
        exp = expected(pats, data, offs)
        assert exp[::3].all()
        check(pats, data, offs)


@pytest.mark.parametrize("variant", ENGINES)
def test_empty_haystacks_and_patterns_longer_than_them(variant):
    pats = [b"abc", b"abcdefgh", b"bcdefghij"]
    hays = [b"", b"ab", b"abc", b"", b"abcdefg", b"bcdefghi", b"xabcx", b"", b"ab" * 2, b"abcdefghij"] + [b""] * 5
    data, offs = batch(hays)
    with forced(variant):
        ac = check(pats, data, offs)
        assert ac.is_match_device(dev(data), dev(offs)).cpu().tolist() == [False, False, True, False, True, False, True, False,
                                                                           False, True] + [False] * 5
        assert ac.is_match_device(dev(np.zeros(0, dtype=np.uint8)), dev(np.zeros(4, dtype=np.int64))).cpu().tolist() == [False] * 3


@pytest.mark.parametrize("variant", ENGINES)
@pytest.mark.parametrize("shift", [0, 1, 255, 511])
def test_pattern_straddling_two_haystacks_does_not_count(variant, shift):
    pats = [b"abcd", b"needle"]
    hays = [b"xxab", b"cdxx", b"xxxnee", b"dlexx", b"a", b"bcd", b"abcd"] * 50
    data, offs = batch(hays)
    with forced(variant):
        ac = check(pats, data, offs, shift=shift)
        got = ac.is_match_device(dev_at(data, shift), dev(offs)).cpu().tolist()
        assert got == [False] * 6 + [True] + ([False] * 6 + [True]) * 49


@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("shift", [0, 3, 200, 509])
def test_matches_at_task_grid_edges(variant, shift):
    """Haystacks whose only occurrence starts or ends at S - 1, S or S + 1 of the 512-byte window grid (every task
    starts on it), and haystacks that start and end on it."""
    T = 512 if variant == "sieve-small-tasks" else 16384
    rng = np.random.default_rng(shift)
    pat = b"qrstuvw"
    pats = [pat, b"zz"]
    hays, pos = [], shift
    for i in range(90):
        n = int(rng.integers(20, 2 * T + 600)) if i % 9 else (-pos) % 512 or 512   # some haystacks end on the grid
        h = bytearray(rng.integers(97, 112, size=n).astype(np.uint8).tobytes())
        if i % 3 != 2 and n > 40:
            delta = [-1, 0, 1][i % 3] + ([0, len(pat)][(i // 3) % 2])   # start (or end) at grid line + delta
            lines = [g for g in range(pos - pos % 512 + 512, pos + n, 512) if pos + 2 <= g - delta and g - delta + len(pat) <= pos + n - 2]
            if lines:
                at = lines[int(rng.integers(0, len(lines)))] - delta - pos
                h[at:at + len(pat)] = pat
        hays.append(bytes(h))
        pos += n
    data, offs = batch(hays)
    with forced(variant):
        exp = expected(pats, data, offs)
        assert exp.sum() > 30
        ac = check(pats, data, offs, shift=shift)
        assert ac._ac.last_stats["task_bytes"] == T


@pytest.mark.parametrize("variant", ["auto", "sieve"])
def test_config_shapes_scaled(variant):
    cases = [W.config2(2000), W.config3(n_patterns=2000, n_lines=20_000), W.config5(n_patterns=5000, n_haystacks=2000)]
    for pats, data, offs in cases:
        pats = [p.encode() if isinstance(p, str) else p for p in pats]
        if variant == "auto":
            check(pats, data, offs)
        else:
            with forced("sieve"):
                ac = check(pats, data, offs)
                assert engine_of(ac) == "sieve"


def test_utf8_str_haystacks():
    rng = np.random.default_rng(5)
    alpha = ["a", "b", "é", "—", "☃", "𝄞"]
    pats = sorted({"".join(rng.choice(alpha, size=int(rng.integers(1, 4)))) for _ in range(12)} - {"a", "b"})
    hays = ["".join(rng.choice(alpha, size=int(rng.integers(0, 12)))) for _ in range(400)]
    exp = [any(p in h for p in pats) for h in hays]
    assert 0 < sum(exp) < len(hays)
    for kind in KINDS:
        ac = AhoCorasick(pats, kind)
        assert ac.is_match_batch(hays) == exp
        assert [ac.is_match(h) for h in hays[:40]] == exp[:40]
        data, offs = batch(hays)
        assert ac.is_match_device(dev(data), dev(offs)).cpu().tolist() == exp


# ---------------------------------------------------------------- the answer does not depend on the match kind
@pytest.mark.parametrize("variant", ENGINES)
def test_match_kinds_give_the_same_mask(variant):
    rng = np.random.default_rng(21)
    pats = sorted({bytes(rng.integers(97, 100, size=int(rng.integers(1, 6))).astype(np.uint8)) for _ in range(15)})
    pats = [p for p in pats if len(p) > 2] + [b"ab"]
    data, offs = W.ragged(200, 30, b"abcx", seed=22)
    with forced(variant):
        masks = []
        for kind in KINDS:
            ac = BytesAhoCorasick(pats, kind)
            m = ac.is_match_device(dev(data), dev(offs)).cpu().tolist()
            hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
            assert m == [len(ac.find_matches_as_indexes(h)) > 0 for h in hays]
            assert m == ac.is_match_batch(hays)
            masks.append(m)
        assert masks[0] == masks[1] == masks[2]
        assert masks[0] == expected(pats, data, offs).tolist()


# ---------------------------------------------------------------- engine selection
def test_engine_follows_the_scan_rule(monkeypatch):
    pats, data, offs = W.config2(1100)   # 4.5 MB of config-2 text: the profile picks the staged table walker
    pats = [p.encode() for p in pats]
    assert data.nbytes >= matcher._Automaton.AUTO_PROFILE_BYTES
    ac = BytesAhoCorasick(pats)
    exp = expected(pats, data, offs)
    check(pats, data, offs, ac=ac)
    assert engine_of(ac) == "table" and ac._ac.last_stats["mode"] == "any"
    monkeypatch.setattr(matcher._Automaton, "ENGINE", "sieve")
    got = ac.is_match_device(dev(data), dev(offs))
    assert engine_of(ac) == "sieve" and np.array_equal(got.cpu().numpy(), exp)


def many_matches_batch():
    """40 haystacks with 200 matches each (8 000: more than the first buffer of a fresh automaton holds), then 60
    haystacks with one match or none: a list cut at the buffer's end would report those as False."""
    hays = [b"x" + b"ab" * 200 for _ in range(40)] + [b"xxabxx" if i % 2 else b"xxxxxx" for i in range(60)]
    return [b"ab", b"zzz"], *batch(hays)


@pytest.mark.parametrize("variant", ["staged", "plain", "global-segments", "engine-table"])
def test_table_walker_async_with_more_matches_than_the_first_buffer(variant, monkeypatch):
    pats, data, offs = many_matches_batch()
    exp = expected(pats, data, offs)
    assert exp[:40].all() and exp[41::2].all() and not exp[40::2].any()
    if variant == "engine-table":   # the tuning knob stays at auto; ENGINE picks the walkers
        monkeypatch.setattr(matcher._Automaton, "ENGINE", "table")
    with contextlib.nullcontext() if variant == "engine-table" else forced(variant):
        for kind in KINDS:
            ac = BytesAhoCorasick(pats, kind)   # fresh: its workspace has the default capacity
            got = ac.is_match_device(dev(data), dev(offs), sync=False)
            torch.cuda.synchronize()
            assert engine_of(ac) == "table"
            assert np.array_equal(got.cpu().numpy(), exp), kind
            out = torch.zeros(len(offs) - 1, dtype=torch.bool, device="cuda")
            out[0] = True
            BytesAhoCorasick(pats, kind).is_match_device(dev(data), dev(offs), out=out, sync=False)
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy(), exp)


def test_two_threads_on_the_table_walker_path(monkeypatch):
    """is_match_device on the walker path reads the automaton's shared workspace: two threads, each on its own
    stream, with batches of different sizes, share one automaton and both get their own answers."""
    monkeypatch.setattr(matcher._Automaton, "ENGINE", "table")
    pats, data0, offs0 = many_matches_batch()
    data1, offs1 = batch([b"ab" if i % 3 == 0 else b"xzzzx" if i % 3 == 1 else b"xyx" for i in range(257)])
    inputs = [(data0, offs0), (data1, offs1)]
    exps = [expected(pats, d, o) for d, o in inputs]
    ac = BytesAhoCorasick(pats)
    errors = []

    def work(t):
        try:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                d, o = dev(inputs[t][0]), dev(inputs[t][1])
                for _ in range(30):
                    got = ac.is_match_device(d, o, sync=bool(t))
                    stream.synchronize()
                    assert np.array_equal(got.cpu().numpy(), exps[t])
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


# ---------------------------------------------------------------- accumulation and the skip counters
@pytest.mark.parametrize("variant", ["sieve", "sieve-small-tasks"])
@pytest.mark.parametrize("shift", [0, 188, 511])
def test_preflagged_haystacks_are_skipped_exactly(variant, shift):
    rng = np.random.default_rng(9)
    n, L = 9, 1 << 20
    data = rng.integers(97, 101, size=n * L, dtype=np.uint8).astype(np.uint8)   # a..d: no pattern occurs
    offs = np.arange(n + 1, dtype=np.int64) * L
    pats = [b"abcz", b"zz", b"dcbaz"]
    ac = BytesAhoCorasick(pats)
    with forced(variant):
        d, o = dev_at(data, shift), dev(offs)
        pre = np.arange(n) % 2 == 0
        out = torch.from_numpy(pre.copy()).cuda()
        ac.is_match_device(d, o, out=out)
        assert out.cpu().numpy().tolist() == pre.tolist()
        st = ac._ac.last_stats
        T = st["task_bytes"]
        assert T == (512 if variant == "sieve-small-tasks" else 16384)
        tasks, windows = predicted_any_skips(d.data_ptr(), offs, pre, T)
        assert (st["tasks_skipped"], st["windows_skipped"]) == (tasks, windows)
        assert tasks > 0 and st["tasks"] == (n * L + (d.data_ptr() & 511) + T - 1) // T
        if shift and T > 512:
            assert windows > 0
        # nothing pre-flagged: nothing skipped, nothing found
        fresh = ac.is_match_device(d, o)
        assert not fresh.any() and ac._ac.last_stats["tasks_skipped"] == ac._ac.last_stats["windows_skipped"] == 0
        # a pre-flagged haystack with matches stays True, one without matches that gets one becomes True
        data2 = data.copy()
        data2[2 * L + 1000:2 * L + 1004] = np.frombuffer(b"abcz", dtype=np.uint8)
        data2[3 * L + 5:3 * L + 7] = np.frombuffer(b"zz", dtype=np.uint8)
        out = torch.from_numpy(pre.copy()).cuda()
        ac.is_match_device(dev_at(data2, shift), o, out=out)
        want = pre.copy()
        want[3] = True
        assert out.cpu().numpy().tolist() == want.tolist()


# ---------------------------------------------------------------- one large haystack: early exit
def test_one_large_haystack_stops_early():
    n = 256 << 20
    ac = BytesAhoCorasick([b"needle", b"haystack"], MatchKind.LeftmostLongest)
    offs = torch.tensor([0, n], dtype=torch.int64, device="cuda")
    hay = torch.full((n,), ord("x"), dtype=torch.uint8, device="cuda")
    with forced("sieve"):
        assert ac.is_match_device(hay, offs).cpu().tolist() == [False]
        st = ac._ac.last_stats
        assert st["tasks_skipped"] == 0 and st["windows_skipped"] == 0 and st["tasks"] >= n // 16384
        hay[700:706] = torch.frombuffer(bytearray(b"needle"), dtype=torch.uint8).cuda()
        assert ac.is_match_device(hay, offs).cpu().tolist() == [True]
        st = ac._ac.last_stats
        assert st["tasks_skipped"] > st["tasks"] // 2, st
        hay[700:706] = ord("x")
        hay[n - 8:] = torch.frombuffer(bytearray(b"haystack"), dtype=torch.uint8).cuda()
        assert ac.is_match_device(hay, offs).cpu().tolist() == [True]
    del hay


# ---------------------------------------------------------------- windows and runs above one call's range
def test_windows_and_runs_match_one_call(monkeypatch):
    rng = np.random.default_rng(31)
    pats = sorted({bytes(rng.integers(97, 101, size=rng.integers(2, 9)).astype(np.uint8)) for _ in range(200)})
    # (a) runs of whole haystacks
    data, offs = W.ragged(400, 3000, b"abcdxyz", seed=32)
    ac = BytesAhoCorasick(pats)
    one = ac.is_match_device(dev(data), dev(offs)).cpu().numpy()
    assert 0 < one.sum() < len(one)
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", 50_000)
    runs = ac.is_match_device(dev(data), dev(offs)).cpu().numpy()
    monkeypatch.undo()
    assert np.array_equal(runs, one) and np.array_equal(one, expected(pats, data, offs))
    # (b) one oversized haystack among small ones; its only occurrence straddles a window edge
    limit, pat = 30_001, b"needle12"
    halo = len(pat) - 1
    step = limit - halo
    big = bytearray(b"x" * 400_000)
    at = 3 * step + limit - 4   # crosses the end of window 3; window 4 holds it whole
    big[at:at + len(pat)] = pat
    hays = [b"xneedle12", b"xx", bytes(big), b"needle1", b"needle12" * 3]
    data, offs = batch(hays)
    ac = BytesAhoCorasick([pat])
    exp = [True, False, True, False, True]
    assert ac.is_match_device(dev(data), dev(offs)).cpu().tolist() == exp
    monkeypatch.setattr(matcher._Automaton, "WINDOW_BYTES", limit)
    with forced("sieve"):
        assert ac.is_match_device(dev(data), dev(offs)).cpu().tolist() == exp
        assert ac.is_match(bytes(big)) is True
        # the windows stop at the first one that sets the flag: a match in the first window costs one launch
        early = bytes(pat) + bytes(big[len(pat):at]) + b"x" * len(pat) + bytes(big[at + len(pat):])
        n0 = _capi.lib().acb_launch_count()
        assert ac.is_match(early) is True
        assert _capi.lib().acb_launch_count() == n0 + 1
        n0 = _capi.lib().acb_launch_count()
        assert ac.is_match(b"x" * 400_000) is False
        assert _capi.lib().acb_launch_count() - n0 == -(-(400_000 - halo) // step)


# ---------------------------------------------------------------- launches, sync=False, threads
def test_one_launch_per_sieve_call_and_async():
    pats, data, offs = W.config3(n_patterns=500, n_lines=2000)
    ac = BytesAhoCorasick(pats)
    exp = expected(pats, data, offs)
    d, o = dev(data), dev(offs)
    with forced("sieve"):
        ac.is_match_device(d, o)
        L = _capi.lib()
        n0 = L.acb_launch_count()
        for _ in range(3):
            got = ac.is_match_device(d, o, sync=False)
        assert L.acb_launch_count() == n0 + 3
        torch.cuda.synchronize()
        assert np.array_equal(got.cpu().numpy(), exp)


def test_two_threads_share_one_automaton():
    rng = np.random.default_rng(41)
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(3, 7))).astype(np.uint8)) for _ in range(60)})
    ac = BytesAhoCorasick(pats)
    inputs = []
    for t in range(2):
        data, offs = W.ragged(300, 200 + 100 * t, b"abcdxyz", seed=50 + t)
        hays = [data[offs[h]:offs[h + 1]].tobytes() for h in range(len(offs) - 1)]
        inputs.append((hays, expected(pats, data, offs).tolist()))
    errors = []

    def work(t):
        try:
            hays, exp = inputs[t]
            for _ in range(25):
                assert ac.is_match_batch(hays) == exp
        except Exception as e:   # noqa: BLE001 -- reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ac.is_match_batch([]) == []
