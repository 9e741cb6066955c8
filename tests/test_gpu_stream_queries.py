"""GPU tests of the stream queries (-m gpu): is_match, find_first and count_matches stream batches and single streams,
compared after every feed with the CPU oracle on each stream's prefix (tests/stream_query_model.expected): ragged
small-alphabet sets in up to 200 slots that start new streams after `last`, at small tasks; code points with chunks cut
inside characters; kilobyte patterns whose tails span several 512-byte tasks; a pending leftmost first match held over
several feeds; a count over more than ACB_LONG_STRETCH records on the grid; agreement with the rows stream; the
is_match skip; argument errors."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind  # noqa: E402
from oracle import Oracle  # noqa: E402

from .gpu_helpers import dev  # noqa: E402
from .stream_model import released_by  # noqa: E402
from .stream_query_model import expected  # noqa: E402
from .test_gpu_stream import b2c, ragged_queues, tuned  # noqa: E402

KINDS = [MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest]
QUERIES = [("is_match", k, False) for k in KINDS] + [("find_first", k, False) for k in KINDS] + \
          [("count", k, False) for k in KINDS] + [("count", MatchKind.Standard, True)]
QUERY_IDS = [f"{q}-{k.name}{'-overlapping' if o else ''}" for q, k, o in QUERIES]


def make_batch(ac, query, n, overlapping):
    if query == "is_match":
        return ac.is_match_stream_batch(n)
    if query == "find_first":
        return ac.find_first_stream_batch(n)
    return ac.count_matches_stream_batch(n, overlapping)


def answer(query, out, i):
    if query == "is_match":
        return bool(out[i])
    if query == "find_first":
        return tuple(int(x) for x in out[i]) if out[i][0] >= 0 else None
    return int(out[i])


def run_queues(ac, pats, query, kind, overlapping, queues, rng, step_max, codepoints=False):
    """Feeds each slot's queue of streams in random steps to a batch of `ac` (a public class), checking every stream's
    answer after every feed."""
    n = len(queues)
    sb = make_batch(ac, query, n, overlapping)
    orc, over = Oracle(pats, kind.name), Oracle(pats, "Standard")
    max_len = max(len(p) for p in pats)
    pos, cur = [0] * n, [0] * n
    done = 0
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
        out = sb.feed_device(dev(data), dev(offs), dev(last) if last.any() else None).cpu().numpy()
        assert sb.last_stats["engine"] == "sieve" and sb.last_stats["mode"] == sb.MODE
        for i in range(n):
            if cur[i] >= len(queues[i]):
                continue
            raw = queues[i][cur[i]]
            want = expected(orc, over, raw[:pos[i]], raw, kind.value, max_len, query, overlapping, bool(last[i]))
            if codepoints and query == "find_first" and want is not None:
                m = b2c(raw)
                want = (want[0], int(m[want[1]]), int(m[want[2]]))
            assert answer(query, out, i) == want, (query, i, cur[i], pos[i])
            if last[i]:
                pos[i] = 0
                cur[i] += 1
                done += 1
    return sb, done


@pytest.mark.parametrize("tuning", ["default", "small-tasks"])
@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
def test_ragged_streams(tuning, query):
    q, kind, overlapping = query
    rng = np.random.default_rng(900 + kind.value + 4 * overlapping + 10 * ["is_match", "find_first", "count"].index(q))
    for shortest in (1, 3):
        pats = sorted({rng.integers(97, 101, size=int(rng.integers(shortest, shortest + 4))).astype(np.uint8).tobytes() for _ in range(30)})
        pats += pats[:2]
        ac = BytesAhoCorasick(pats, kind)
        with tuned(tuning):
            for n in (1, 7, 200):
                _, done = run_queues(ac, pats, q, kind, overlapping, ragged_queues(rng, n, pats, shortest), rng, step_max=3 * shortest + 6)
                assert done >= 1


@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
def test_code_points_cut_inside_characters(query):
    q, kind, overlapping = query
    rng = np.random.default_rng(40 + kind.value + 4 * overlapping)
    alphabet = ["a", "b", "é", "ж", "€", "中", "😀", "𝄞"]
    pats_s = sorted({"".join(rng.choice(alphabet, size=int(rng.integers(1, 5)))) for _ in range(30)})
    pats = [p.encode() for p in pats_s]
    ac = AhoCorasick(pats_s, kind)
    queues = []
    for i in range(60):
        text = "".join(rng.choice(alphabet, size=int(rng.integers(0, 120))))
        if text and i % 3 == 0:
            at = int(rng.integers(0, len(text) + 1))
            text = text[:at] + pats_s[i % len(pats_s)] * 2 + text[at:]
        queues.append([text.encode(), "ab€".encode() * 5])
    run_queues(ac, pats, q, kind, overlapping, queues, rng, step_max=7, codepoints=True)
    # the single-stream object takes str chunks; its answers are the one-shot calls on the prefix / the whole text
    text = "".join(rng.choice(alphabet, size=300))
    s = {"is_match": ac.is_match_stream, "find_first": ac.find_first_stream}.get(q, lambda: ac.count_matches_stream(overlapping))()
    for a in range(0, 300, 17):
        got = s.feed(text[a:a + 17])
        if q == "is_match":
            assert got == ac.is_match(text[:a + 17])
    final = s.finish()
    whole = {"is_match": lambda: ac.is_match(text), "find_first": lambda: ac.find_first(text),
             "count": lambda: ac.count_matches(text, overlapping)}[q]()
    assert final == whole


@pytest.mark.parametrize("tuning", ["default", "small-tasks"])
@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
def test_kilobyte_patterns(tuning, query):
    """Patterns of 300 to 3 000 bytes: the tail spans several 512-byte tasks."""
    q, kind, overlapping = query
    rng = np.random.default_rng(600 + kind.value + 4 * overlapping)
    base = [rng.integers(97, 101, size=int(rng.integers(300, 3001))).astype(np.uint8).tobytes() for _ in range(12)]
    pats = base + [b[:len(b) // 2] for b in base[:4]] + [b[len(b) // 3:] for b in base[4:8]] + base[:1]
    queues = []
    for i in range(8):
        parts = []
        for _ in range(4):
            parts.append(rng.integers(97, 101, size=int(rng.integers(0, 2000))).astype(np.uint8).tobytes())
            parts.append(pats[int(rng.integers(0, len(pats)))] if rng.random() < 0.7 else base[int(rng.integers(0, 12))][:250])
        queues.append([b"".join(parts)])
    ac = BytesAhoCorasick(pats, kind)
    with tuned(tuning):
        for step_max in (200, 6000):
            run_queues(ac, pats, q, kind, overlapping, queues, rng, step_max=step_max)


@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_a_pending_leftmost_first_match_is_held_over_several_feeds(kind):
    """A 40-byte pattern whose prefix "x" is a pattern too: once "x" is seen the candidate stays pending (its chunk
    scans skipped) until 40 bytes past its start are fed; the long pattern, if it completes, wins under both kinds
    only for LeftmostLongest (LeftmostFirst: the lower index, "x" = 0, at the same start)."""
    long_pat = b"x" + b"y" * 39
    ac = BytesAhoCorasick([b"x", long_pat], kind)
    s = ac.find_first_stream()
    assert s.feed(b"ab") is None
    assert s.feed(b"cx") is None and s.last_stats["pending"] == 1
    for _ in range(4):
        assert s.feed(b"y" * 9) is None and s.last_stats["pending"] == 1
    got = s.feed(b"y" * 9)   # 3 + 45 = 48 bytes fed > 3 + 40
    want = (1, 3, 43) if kind == MatchKind.LeftmostLongest else (0, 3, 4)
    assert got == want and s.last_stats["pending"] == 0
    assert s.finish() == want
    s = ac.find_first_stream()
    assert s.feed(b"zzx") is None and s.feed(b"yy") is None
    assert s.finish() == (0, 2, 3)   # the stream ended: the pending candidate is final


def test_non_overlapping_count_on_the_grid():
    """One stream whose sequences exceed ACB_LONG_STRETCH records: counted on the whole grid, equal to the oracle."""
    rng = np.random.default_rng(3)
    pats = [b"ab", b"abab", b"ba", b"b", b"aba"]
    raw = rng.integers(97, 99, size=300_000).astype(np.uint8).tobytes()
    for kind in KINDS:
        ac = BytesAhoCorasick(pats, kind)
        sb = ac.count_matches_stream_batch(2)
        orc = Oracle(pats, kind.name)
        full = orc.find(raw)
        cut = [0, 70_001, 70_003, 200_000, len(raw)]
        for a, b in zip(cut, cut[1:]):
            last = b == len(raw)
            data = np.frombuffer(raw[a:b] * 2, dtype=np.uint8)
            offs = np.array([0, b - a, 2 * (b - a)], dtype=np.int64)
            out = sb.feed_device(dev(data), dev(offs), dev(np.array([last, last]))).cpu().tolist()
            want = len(released_by(full, b, kind.value, False, 4, last))
            assert out == [want, want]
            if b - a > 100_000:
                assert sb.last_stats["long_stretches"] == 2
        assert out == [len(full)] * 2 == [ac.count_matches(raw)] * 2


@pytest.mark.parametrize("kind", KINDS)
def test_agreement_with_the_rows_stream(kind):
    """The same chunks fed to the rows stream: count = the rows released so far, find_first = the first released row."""
    rng = np.random.default_rng(kind.value)
    pats = sorted({rng.integers(97, 100, size=int(rng.integers(2, 6))).astype(np.uint8).tobytes() for _ in range(20)})
    ac = BytesAhoCorasick(pats, kind)
    raw = rng.integers(97, 100, size=20_000).astype(np.uint8).tobytes()
    rows_s, cnt_s, first_s = ac.stream(), ac.count_matches_stream(), ac.find_first_stream()
    released = []
    for a in range(0, len(raw), 777):
        c = raw[a:a + 777]
        released += rows_s.feed(c)
        assert cnt_s.feed(c) == len(released)
        f = first_s.feed(c)
        assert f == (tuple(released[0]) if released else None)
    released += rows_s.finish()
    assert cnt_s.finish() == len(released) and first_s.finish() == tuple(released[0])


def test_is_match_streams_skip_their_chunks_once_flagged():
    """4 096 streams whose first feed matches: every later feed's chunk tasks are skipped."""
    ac = BytesAhoCorasick([b"needle"])
    n, per = 4096, 16 << 10
    sb = ac.is_match_stream_batch(n)
    data = torch.full((n * per,), ord("a"), dtype=torch.uint8, device="cuda")
    offs = torch.arange(0, n + 1, dtype=torch.int64, device="cuda") * per
    data.view(n, per)[:, 100:106] = torch.tensor(list(b"needle"), dtype=torch.uint8, device="cuda")
    assert bool(sb.feed_device(data, offs).all())
    data.view(n, per)[:, 100:106] = ord("a")
    out = sb.feed_device(data, offs)
    assert bool(out.all()) and sb.last_stats["tasks_skipped"] > 0 and sb.last_stats["flagged"] == n
    last = torch.zeros(n, dtype=torch.bool, device="cuda")
    last[::2] = True
    assert bool(sb.feed_device(data, offs, last).all())
    out = sb.feed_device(data, offs).cpu()   # the ended streams start again, with no match
    assert out[1::2].all() and not out[::2].any()


def test_argument_errors():
    ac = BytesAhoCorasick([b"ab"])
    for sb in (ac.is_match_stream_batch(2), ac.find_first_stream_batch(2), ac.count_matches_stream_batch(2)):
        data = torch.zeros(4, dtype=torch.uint8, device="cuda")
        with pytest.raises(TypeError, match="offsets"):
            sb.feed_device(data, torch.zeros(2, dtype=torch.int64, device="cuda"))
        with pytest.raises(TypeError, match="offsets"):
            sb.feed_device(data, torch.zeros(3, dtype=torch.int32, device="cuda"))
        offs = torch.tensor([0, 2, 4], dtype=torch.int64, device="cuda")
        with pytest.raises(TypeError, match="last"):
            sb.feed_device(data, offs, torch.zeros(2, dtype=torch.uint8, device="cuda"))
        with pytest.raises(TypeError, match="last"):
            sb.feed_device(data, offs, torch.zeros(3, dtype=torch.bool, device="cuda"))
        sb.feed_device(data, offs)
    with pytest.raises(ValueError, match="overlapping"):
        BytesAhoCorasick([b"ab"], MatchKind.LeftmostFirst).count_matches_stream(overlapping=True)
    s = ac.count_matches_stream()
    assert s.feed(b"xa") == 0 and s.feed(b"bab") == 2 and s.finish() == 2
    with pytest.raises(RuntimeError, match="feed after finish"):
        s.feed(b"ab")
    s = AhoCorasick(["ab"]).is_match_stream()
    assert s.feed("xa") is False and s.feed("b") is True and s.finish() is True
