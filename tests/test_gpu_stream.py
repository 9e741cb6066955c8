"""GPU tests of the stream search (-m gpu): StreamBatch.feed_device and the single-stream objects, compared with the CPU
oracle on each stream's concatenation after its last feed, and with the release rule's prefix of that result after
every feed.  Ragged small-alphabet sets split among 1 to 300 streams with random per-feed chunk lengths (empty chunks,
streams ending with `last` and reused), at small tasks and forced sieve rings; code points with chunks cut inside
characters; long patterns; positions past 2^32; config 3 and config 4 at size against scan_device; two threads."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi, matcher  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, dev  # noqa: E402
from .stream_model import released_by  # noqa: E402

# name -> acb_set_tuning(kernel, hot_rows, segment_bytes, table, sieve_ring)
TUNINGS = {"default": (0, 0, 0, 0, 0), "small-tasks": (5, 0, 512, 0, 0), "ring-1": (5, 0, 512, 0, 1), "ring-2": (5, 0, 0, 0, 2)}


class tuned:
    def __init__(self, name):
        self.t = TUNINGS[name]

    def __enter__(self):
        _capi.set_tuning(*self.t)

    def __exit__(self, *exc):
        _capi.set_tuning()


def b2c(raw: bytes):
    """byte offset -> code point index, for every offset 0 .. len(raw) (continuation bytes counted before it)."""
    a = np.frombuffer(raw, dtype=np.uint8)
    cont = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum((a & 0xC0) == 0x80, out=cont[1:])
    return np.arange(len(raw) + 1) - cont


class Driver:
    """Feeds per-stream byte strings to a StreamBatch in random steps and checks every feed.  Each slot runs a queue of
    streams: when one ends (with `last`) the slot starts the next."""

    def __init__(self, ac, pats, kind, overlapping, codepoints=False):
        self.ac, self.kind, self.overlapping, self.codepoints = ac, kind, overlapping, codepoints
        self.orc = Oracle(pats, kind.name)
        self.max_len = max(len(p) for p in pats)
        self.pats = pats

    def expected(self, raw):
        return self.orc.find(raw, overlapping=self.overlapping)

    def run(self, queues, rng, step_max, sb=None):
        n = len(queues)
        sb = sb or matcher.StreamBatch(self.ac, n, self.overlapping, self.codepoints)
        pos = [0] * n                # bytes of the current stream fed
        cur = [0] * n                # index of the current stream in each queue
        got = [[] for _ in range(n)]
        streams_done = 0
        while any(c < len(q) for c, q in zip(cur, queues)):
            chunks, last = [], np.zeros(n, dtype=bool)
            for i in range(n):
                if cur[i] >= len(queues[i]):
                    chunks.append(b"")
                    continue
                raw = queues[i][cur[i]]
                k = 0 if rng.random() < 0.15 else int(rng.integers(1, step_max + 1))
                chunks.append(raw[pos[i]:pos[i] + k])
                pos[i] = min(len(raw), pos[i] + k)
                last[i] = pos[i] == len(raw) and rng.random() < 0.7
            offs = np.zeros(n + 1, dtype=np.int64)
            np.cumsum([len(c) for c in chunks], out=offs[1:])
            data = np.frombuffer(b"".join(chunks) or b"\0", dtype=np.uint8)[: offs[-1]]
            rows, ro = sb.feed_device(dev(data), dev(offs), dev(last) if last.any() else None)
            rows, ro = rows.cpu().numpy(), ro.cpu().numpy()
            assert ro[0] == 0 and ro[-1] == len(rows) and np.all(np.diff(ro) >= 0)
            st = sb.last_stats
            assert st["mode"] == "stream" and st["engine"] == "sieve" and st["released"] == len(rows)
            for i in range(n):
                if cur[i] >= len(queues[i]):
                    assert ro[i + 1] == ro[i]
                    continue
                part = rows[ro[i]:ro[i + 1]]
                assert np.all(part[:, 0] == i)
                got[i] += [tuple(r) for r in part[:, 1:].tolist()]
                raw = queues[i][cur[i]]
                full = self.expected(raw)
                want = released_by(full, pos[i], self.kind.value, self.overlapping, self.max_len, bool(last[i]))
                if self.codepoints:
                    m = b2c(raw)
                    want = [(p, int(m[s]), int(m[e])) for p, s, e in want]
                    text = raw.decode("utf-8")
                    for p, s, e in got[i]:
                        assert text[s:e] == self.pats[p].decode("utf-8")
                assert got[i] == want, (i, cur[i], pos[i])
                if last[i]:
                    got[i], pos[i] = [], 0
                    cur[i] += 1
                    streams_done += 1
        return sb, streams_done


def ragged_queues(rng, n, pats, shortest, per_slot=2):
    queues = []
    for i in range(n):
        q = []
        for _ in range(per_slot):
            h = rng.integers(97, 101, size=int(rng.integers(0, 40 * shortest + 1))).astype(np.uint8).tobytes() if rng.random() > 0.05 else b""
            if h and rng.random() < 0.5:
                at = int(rng.integers(0, len(h) + 1))
                h = h[:at] + pats[int(rng.integers(0, len(pats)))] * 3 + h[at:]
            q.append(h)
        queues.append(q)
    return queues


def small_alphabet_patterns(rng, shortest):
    pats = sorted({bytes(rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 7))).astype(np.uint8)) for _ in range(40)})
    return pats + pats[:2]   # duplicates: distinct ids, same bytes


@pytest.mark.parametrize("tuning", list(TUNINGS))
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("shortest", [1, 3, 9])
def test_ragged_streams(tuning, search, shortest):
    kind, overlapping = search
    rng = np.random.default_rng(900 + 10 * shortest + kind.value + 4 * overlapping)
    pats = small_alphabet_patterns(rng, shortest)
    ac = BytesAhoCorasick(pats, kind)
    drv = Driver(ac._ac, pats, kind, overlapping)
    with tuned(tuning):
        for n in (1, 37, 300):
            queues = ragged_queues(rng, n, pats, shortest)
            _, done = drv.run(queues, rng, step_max=int(rng.choice([1, 5, 3 * shortest + 10, 200])))
            assert done >= 1


def test_one_byte_patterns_and_the_issue_example():
    """max_pattern_len == 1 (no tail), and the example of the contract: abcd / bc, LeftmostLongest."""
    rng = np.random.default_rng(5)
    for search in SEARCHES:
        kind, overlapping = search
        pats = [b"a", b"b", b"a"]
        drv = Driver(BytesAhoCorasick(pats, kind)._ac, pats, kind, overlapping)
        drv.run(ragged_queues(rng, 20, pats, 1), rng, step_max=4)
    ac = BytesAhoCorasick([b"abcd", b"bc"], MatchKind.LeftmostLongest)
    s = ac.stream()
    assert s.feed(b"xab") == [] and s.last_stats["held"] == 0   # no candidate yet
    assert s.feed(b"cd") == [(0, 1, 5)]
    assert s.finish() == []
    with pytest.raises(RuntimeError):
        s.feed(b"x")
    s = ac.stream()
    assert s.feed(b"xabc") == [] and s.last_stats["held"] == 1   # bc (1, 2, 4) is pending: abcd may still come
    # released; the restart point (5) now lies past the new tail's start (2): the next feed's selection resumes there
    assert s.feed(b"d") == [(0, 1, 5)] and s.last_stats["held"] == 1
    assert s.finish() == [] and s.last_stats["held"] == 0


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_code_points_cut_inside_characters(search):
    kind, overlapping = search
    rng = np.random.default_rng(40 + kind.value + 4 * overlapping)
    alphabet = ["a", "b", "é", "ж", "€", "中", "😀", "𝄞"]   # 1- to 4-byte characters
    pats_s = sorted({"".join(rng.choice(alphabet, size=int(rng.integers(1, 5)))) for _ in range(30)})
    pats = [p.encode() for p in pats_s]
    ac = AhoCorasick(pats_s, kind)
    drv = Driver(ac._ac, pats, kind, overlapping, codepoints=True)
    queues = []
    for i in range(60):
        text = "".join(rng.choice(alphabet, size=int(rng.integers(0, 120))))
        if text and i % 3 == 0:
            at = int(rng.integers(0, len(text) + 1))
            text = text[:at] + pats_s[i % len(pats_s)] * 2 + text[at:]
        queues.append([text.encode()])
    drv.run(queues, rng, step_max=7)   # byte steps: most cuts fall inside characters
    # the single-stream object takes str chunks
    s = ac.stream(overlapping)
    text = "".join(rng.choice(alphabet, size=300))
    got = []
    for a in range(0, 300, 17):
        got += s.feed(text[a:a + 17])
    got += s.finish()
    assert got == Oracle(pats, kind.name).find_str(text, overlapping=overlapping)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_long_patterns(search):
    """The reference benchmark's names (4 244, 221 duplicates): the tail is as long as the longest name."""
    kind, overlapping = search
    rng = np.random.default_rng(77)
    pats_s = W.patterns_long()
    pats = [p.encode() for p in pats_s]
    ac = AhoCorasick(pats_s, kind)
    drv = Driver(ac._ac, pats, kind, overlapping, codepoints=True)
    queues = []
    for i in range(24):
        words = [pats_s[int(j)] if rng.random() < 0.3 else "notaperson" for j in rng.integers(0, len(pats_s), size=60)]
        queues.append([" ".join(words).encode()])
    drv.run(queues, rng, step_max=max(len(p) for p in pats) + 50)


@pytest.mark.parametrize("tuning", ["default", "small-tasks"])
@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_kilobyte_patterns(tuning, search):
    """Patterns of 300 to 3 000 bytes (and prefixes and suffixes of them, so the leftmost kinds choose), planted in
    random text: the tail is kilobytes, longer than a sieve task at 512-byte tasks, and chunks are both shorter and
    longer than it."""
    kind, overlapping = search
    rng = np.random.default_rng(600 + kind.value + 4 * overlapping)
    base = [rng.integers(97, 101, size=int(rng.integers(300, 3001))).astype(np.uint8).tobytes() for _ in range(12)]
    pats = base + [b[:len(b) // 2] for b in base[:4]] + [b[len(b) // 3:] for b in base[4:8]] + base[:1]
    queues = []
    for i in range(8):
        parts = []
        for _ in range(6):
            parts.append(rng.integers(97, 101, size=int(rng.integers(0, 2000))).astype(np.uint8).tobytes())
            parts.append(pats[int(rng.integers(0, len(pats)))] if rng.random() < 0.8 else base[int(rng.integers(0, 12))][:250])
        queues.append([b"".join(parts)])
    drv = Driver(BytesAhoCorasick(pats, kind)._ac, pats, kind, overlapping)
    assert drv.max_len > 2000
    with tuned(tuning):
        for step_max in (200, 6000):
            drv.run(queues, rng, step_max=step_max)


def test_positions_past_2_to_the_32():
    """One stream fed five 1 GiB chunks; patterns planted across the chunk seams and around byte 2^32."""
    pats = [b"needle", b"haystackseam", b"ok"]
    chunk_bytes = 1 << 30
    plants = [(1, k * chunk_bytes - 5) for k in range(1, 5)]   # across each seam; the last one across byte 2^32
    plants += [(2, (1 << 32) - 20), (0, (1 << 32) + 50), (0, (1 << 32) + 100), (0, 5 * chunk_bytes - 6)]
    buf = torch.zeros(chunk_bytes, dtype=torch.uint8, device="cuda")
    for search in [(MatchKind.Standard, True), (MatchKind.LeftmostLongest, False)]:
        kind, overlapping = search
        s = BytesAhoCorasick(pats, kind).stream_batch(1, overlapping)
        got = []
        for k in range(5):
            buf.zero_()
            lo = k * chunk_bytes
            for pid, at in plants:
                p = pats[pid]
                for j, b in enumerate(p):
                    if lo <= at + j < lo + chunk_bytes:
                        buf[at + j - lo] = b
            offs = torch.tensor([0, chunk_bytes], dtype=torch.int64, device="cuda")
            last = torch.tensor([k == 4], device="cuda")
            rows, _ = s.feed_device(buf, offs, last)
            got += [tuple(r) for r in rows[:, 1:].cpu().tolist()]
        want = sorted(((pid, at, at + len(pats[pid])) for pid, at in plants), key=lambda r: (r[2], r[1], r[0]))
        assert got == want
        assert want[-1][2] > 1 << 32


def test_config3_as_1024_streams():
    """Config 3's log lines (512 MiB) as 1 024 streams of 512 KiB, fed in uneven steps of about 256 KiB per stream,
    LeftmostLongest: each stream's rows equal scan_device over the same bytes laid out as 1 024 haystacks."""
    pats, data, offs = W.config3(n_lines=1 << 21)
    n = 1024
    per = len(data) // n
    ac = BytesAhoCorasick(pats, MatchKind.LeftmostLongest)
    d = dev(data[: n * per])
    hoffs = torch.arange(n + 1, dtype=torch.int64, device="cuda") * per
    m, mo, _ = ac.scan_device(d, hoffs)
    want = m.to(torch.int64).cpu().numpy()
    sb = ac.stream_batch(n)
    rng = np.random.default_rng(3)
    fed, parts = 0, []
    while fed < per:
        step = min(per - fed, int(rng.integers(200_000, 320_000)))
        chunk = d.view(n, per)[:, fed:fed + step].reshape(-1)
        o = torch.arange(n + 1, dtype=torch.int64, device="cuda") * step
        last = torch.full((n,), fed + step == per, dtype=torch.bool, device="cuda")
        rows, ro = sb.feed_device(chunk, o, last)
        parts.append((rows.cpu().numpy(), ro.cpu().numpy()))
        fed += step
    got = np.concatenate([np.concatenate([r[ro[i]:ro[i + 1]] for r, ro in parts]) for i in range(n)])
    assert np.array_equal(got, want)


def test_config4_one_overlapping_stream_in_uneven_chunks():
    """Config 4's patterns, one 1 GiB stream fed in 7 uneven chunks, overlapping: the rows equal scan_device on the
    whole buffer."""
    pats = W.random_lowercase_patterns(100_000, 5, 8, 4)
    g = torch.Generator(device="cuda")
    g.manual_seed(4)
    d = torch.randint(97, 123, (1 << 30,), dtype=torch.uint8, device="cuda", generator=g)
    ac = BytesAhoCorasick(pats)
    m, _, _ = ac.scan_device(d, torch.tensor([0, d.numel()], dtype=torch.int64, device="cuda"), True)
    want = m.to(torch.int64)[:, 1:].clone()
    cuts = [0, 1, 7, 100 << 20, 101 << 20, 600 << 20, (600 << 20) + 3, 1 << 30]
    sb = ac.stream_batch(1, overlapping=True)
    got = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        rows, _ = sb.feed_device(d[a:b], torch.tensor([0, b - a], dtype=torch.int64, device="cuda"),
                                 torch.tensor([b == cuts[-1]], device="cuda"))
        got.append(rows[:, 1:].clone())
    assert torch.equal(torch.cat(got), want)


def test_two_threads_and_a_scan_share_one_automaton():
    rng = np.random.default_rng(11)
    pats = small_alphabet_patterns(rng, 3)
    kind = MatchKind.LeftmostFirst
    ac = BytesAhoCorasick(pats, kind)
    errors = []

    def feeder(seed):
        try:
            r = np.random.default_rng(seed)
            drv = Driver(ac._ac, pats, kind, False)
            for _ in range(4):
                drv.run(ragged_queues(r, 50, pats, 3), r, step_max=60)
        except Exception as e:   # reported by the main thread
            errors.append(e)

    def scanner():
        try:
            data, offs = np.frombuffer(b"abcd" * 5000, dtype=np.uint8), np.array([0, 7000, 20000], dtype=np.int64)
            want = Oracle(pats, kind.name).scan_batch(data, offs)[2]
            for _ in range(20):
                m, _, _ = ac.scan_device(dev(data), dev(offs))
                assert np.array_equal(m.cpu().numpy().view(np.uint32), want)
        except Exception as e:
            errors.append(e)

    ts = [threading.Thread(target=feeder, args=(s,)) for s in (1, 2)] + [threading.Thread(target=scanner)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
