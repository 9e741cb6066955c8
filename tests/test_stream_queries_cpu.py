"""CPU tests of the stream queries (is_match, find_first and count_matches per stream): the Python model of the device
design (tests/stream_query_model.py) equals the oracle on each prefix after every feed, on thousands of seeded cases,
with slots that start a new stream after `last`; the grid-marking count with ACB_LONG_STRETCH patched small and the
order inside each round shuffled; the three C entry points refuse bad arguments before any CUDA call; the public
objects validate their arguments before any device work."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from . import stream_query_model as sqm
from .stream_model import KIND_NAMES

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
QUERIES = [("is_match", k, False) for k in range(3)] + [("find_first", k, False) for k in range(3)] + \
          [("count", k, False) for k in range(3)] + [("count", 0, True)]
QUERY_IDS = [f"{q}-{KIND_NAMES[k]}{'-overlapping' if o else ''}" for q, k, o in QUERIES]


def make_model(query, pats, kind, overlapping, over, seed=0):
    if query == "is_match":
        return sqm.IsMatchModel(pats, kind, over)
    if query == "find_first":
        return sqm.FindFirstModel(pats, kind, over)
    return sqm.CountModel(pats, kind, overlapping, over, seed)


def run_slot(query, pats, kind, overlapping, streams, seed=0):
    """One slot fed a queue of streams (each a list of chunks), the last chunk of each with `last`: the model's answer
    equals the oracle's after every feed.  -> the model (its counters)."""
    over = Oracle(pats, "Standard")
    orc = Oracle(pats, KIND_NAMES[kind])
    m = make_model(query, pats, kind, overlapping, over, seed)
    max_len = max(len(p) for p in pats)
    for chunks in streams:
        final = b"".join(chunks)
        prefix = b""
        for i, c in enumerate(chunks):
            last = i == len(chunks) - 1
            prefix += c
            got = m.feed(c, last)
            want = sqm.expected(orc, over, prefix, final, kind, max_len, query, overlapping, last)
            assert got == want, (query, pats, chunks, i)
        assert m.fed == 0 and m.tail == b""
    return m


def random_chunks(rng, hay, max_len):
    cuts, at = [], 0
    while at < len(hay):
        r = rng.random()
        step = 0 if r < 0.1 else 1 if r < 0.25 else max(max_len - 1, 0) + int(rng.integers(-1, 2)) if r < 0.6 else int(rng.integers(1, 3 * max_len + 8))
        at = min(len(hay), at + max(step, 0))
        cuts.append(at)
    return [hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])]


def random_case(rng, shortest):
    pats = sorted({bytes(rng.integers(97, 100, size=int(rng.integers(shortest, shortest + 5))).astype(np.uint8)) for _ in range(12)})
    pats += pats[:1]   # a duplicate: distinct ids, same bytes
    hay = bytearray(rng.integers(97, 100, size=int(rng.integers(0, 120))).astype(np.uint8).tobytes())
    for _ in range(int(rng.integers(0, 4))):
        at = int(rng.integers(0, len(hay) + 1))
        hay[at:at] = pats[int(rng.integers(0, len(pats)))]
    return pats, bytes(hay)


@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
def test_model_equals_the_oracle_on_seeded_cases(query):
    q, kind, overlapping = query
    rng = np.random.default_rng(11 + kind + 10 * overlapping + 100 * ["is_match", "find_first", "count"].index(q))
    for case in range(300):
        pats, _ = random_case(rng, 1 + case % 6)
        max_len = max(len(p) for p in pats)
        streams = []
        for _ in range(3):   # three streams in one slot: `last` ends each, the slot starts again
            _, hay = random_case(rng, 1 + case % 6)
            hay = hay.replace(b"c", b"") + pats[int(rng.integers(0, len(pats)))] if rng.random() < 0.5 else hay
            streams.append(random_chunks(rng, hay, max_len))
        run_slot(q, pats, kind, overlapping, streams)


@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
def test_cuts_at_every_offset_inside_planted_patterns(query):
    q, kind, overlapping = query
    pats = [b"abcd", b"bc", b"cdxyz", b"x", b"zab"]
    hay = b"qqabcdxyzabcdqq"
    for a in range(len(hay) + 1):
        for b in range(a, len(hay) + 1):
            run_slot(q, pats, kind, overlapping, [[hay[:a], hay[a:b], hay[b:]], [b"", hay[a:]]])


@pytest.mark.parametrize("query", QUERIES, ids=QUERY_IDS)
@pytest.mark.parametrize("pats", [[b"a", b"aa", b"aaa"], [b"a", b"b"], [b"aba", b"ab", b"ba", b"aba"]], ids=["nested", "single-byte", "self-overlap"])
def test_nested_self_overlapping_and_one_byte_patterns(query, pats):
    q, kind, overlapping = query
    rng = np.random.default_rng(len(pats))
    for _ in range(100):
        streams = []
        for _ in range(2):
            hay = rng.integers(97, 99, size=int(rng.integers(0, 40))).astype(np.uint8).tobytes()
            cuts = sorted(int(x) for x in rng.integers(0, len(hay) + 1, size=int(rng.integers(0, 8))))
            streams.append([hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])])
        run_slot(q, pats, kind, overlapping, streams)


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_grid_count_with_a_small_long_stretch_and_shuffled_rounds(kind, monkeypatch):
    """Non-overlapping counts of sequences longer than ACB_LONG_STRETCH (patched to 3) take the grid path: successors,
    marks by pointer jumping in shuffled order, release by the rule.  They equal the oracle after every feed."""
    monkeypatch.setattr(sqm, "LONG_STRETCH", 3)
    rng = np.random.default_rng(40 + kind)
    long_total = 0
    for case in range(300):
        pats, hay = random_case(rng, 1 + case % 4)
        hay = hay * 2
        streams = [random_chunks(rng, hay, max(len(p) for p in pats)), [hay]]
        long_total += run_slot("count", pats, kind, False, streams, seed=case).long_stretches
    assert long_total > 100


def test_find_first_skips_the_chunk_of_a_pending_leftmost_candidate():
    """LeftmostLongest abcd / bc: after "xab" nothing is known; "c" makes "bc" (1, 3) a candidate that "abcd" (start 1)
    may still beat, so it is pending and the next chunk's scan is skipped; "d" makes "abcd" the final answer."""
    m = sqm.FindFirstModel([b"abcd", b"bc"], 2)
    assert m.feed(b"xab") is None and m.chunk_scans == 1
    assert m.feed(b"c") is None and m.state[0] == "pending" and m.chunk_scans == 2
    assert m.feed(b"dzzzz") == (0, 1, 5) and m.chunk_scans == 2
    assert m.feed(b"", True) == (0, 1, 5) and m.state is None


# ---------------------------------------------------------------- C entry points
def _automaton(kind=0, pats=(b"hello", b"world")):
    L = _capi.lib()
    offs = np.zeros(len(pats) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pats], out=offs[1:])
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pats), kind, -1, C.byref(h)) == 0
    return L, h


def _advance(L, h, data=FAKE, offs=FAKE, n=1, total=16, last=None, codepoints=0, carry=FAKE, tail=FAKE, seam=FAKE, seam_offs=FAKE,
             scratch=FAKE):
    return L.acb_stream_advance(h, data, offs, n, total, last, codepoints, carry, tail, seam, seam_offs, scratch, None)


def _first(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, last=None, codepoints=0, seam_bytes=16, **ptrs):
    names = ["carry", "seam", "seam_offs"]
    after = ["seam_keys", "chunk_keys", "best", "scratch", "rows"]
    return L.acb_stream_first_resolve(h, sieve, data, offs, n, total, last, codepoints, *[ptrs.get(k, FAKE) for k in names], seam_bytes,
                                      *[ptrs.get(k, FAKE) for k in after], None)


COUNT_PTRS = ["carry", "seam_offs", "seam_list", "seam_mo", "chunk_list", "chunk_mo", "chunk_counts", "running", "counts", "scratch"]


def _count(L, h, data=FAKE, offs=FAKE, n=1, total=16, last=None, overlapping=0, words=1 << 20, **ptrs):
    return L.acb_stream_count(h, data, offs, n, total, last, overlapping, *[ptrs.get(k, FAKE) for k in COUNT_PTRS], words, None)


def test_entry_points_reject_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        common = [(dict(offs=None), "null argument"), (dict(data=None), "null argument"), (dict(n=-1), "n_streams out of range"),
                  (dict(n=0xffffffff), "n_streams out of range"), (dict(total=1 << 31), "must be below 2^31")]
        advance = common + [({k: None}, "null argument") for k in ("carry", "tail", "seam", "seam_offs")] + [
            (dict(codepoints=1, scratch=None), "null argument")]
        for kw, msg in advance:
            assert _advance(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        first = common + [({k: None}, "null argument") for k in ("carry", "seam", "seam_offs", "seam_keys", "chunk_keys", "best", "scratch",
                                                                   "rows")] + [
            (dict(sieve=None), "null argument"), (dict(seam_bytes=1 << 31), "must be below 2^31"),
            (dict(), "acb_sieve_build has not been called")]
        for kw, msg in first:
            assert _first(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        count = common + [({k: None}, "null argument") for k in COUNT_PTRS if k not in ("chunk_counts",)] + [
            (dict(overlapping=1, chunk_counts=None), "null argument"), (dict(overlapping=2), "overlapping must be 0 or 1"),
            (dict(words=4 + 6 * 1 - 1), "dev_scratch is too small"), (dict(overlapping=1, words=3), "dev_scratch is too small")]
        for kw, msg in count:
            assert _count(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_stream_advance(None, FAKE, FAKE, 1, 16, None, 0, FAKE, FAKE, FAKE, FAKE, FAKE, None) == _capi.ACB_EINVAL
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


def test_one_byte_patterns_need_no_tail_or_seam_buffers():
    L, h = _automaton(0, (b"a", b"b"))
    try:
        assert _advance(L, h, tail=None, seam=None, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
        assert _first(L, h, seam=None, seam_bytes=0, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2])
def test_count_refuses_overlapping_on_a_leftmost_automaton(kind):
    L, h = _automaton(kind)
    try:
        assert _count(L, h, overlapping=1) == _capi.ACB_EUNSUPPORTED
        assert f"match kind {KIND_NAMES[kind]} does not support overlapping searches" in _capi.last_error()
    finally:
        L.acb_free(h)


# ---------------------------------------------------------------- Python validation (no device needed)
@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_overlapping_count_on_a_leftmost_automaton_is_refused_at_creation(kind):
    msg = f"match kind {kind.name} does not support overlapping searches"
    for ac in (AhoCorasick(["ab"], kind), BytesAhoCorasick([b"ab"], kind)):
        with pytest.raises(ValueError, match=msg):
            ac.count_matches_stream(overlapping=True)
        with pytest.raises(ValueError, match=msg):
            ac.count_matches_stream_batch(4, overlapping=True)
        ac.count_matches_stream_batch(4)   # non-overlapping: every kind


def test_query_batches_share_the_stream_limits():
    ac = BytesAhoCorasick([b"a" * 1025])
    fits = ac._ac.WINDOW_BYTES // (2 * 1024)
    for make in (ac.is_match_stream_batch, ac.find_first_stream_batch, ac.count_matches_stream_batch):
        sb = make(fits)
        assert sb.n_streams == fits and sb.device is None
        with pytest.raises(ValueError, match="seam bytes"):
            make(fits + 1)
        for bad in ("4", 4.0, True, None):
            with pytest.raises(TypeError):
                make(bad)
        with pytest.raises(ValueError):
            make(-1)


def test_query_batch_argument_types():
    torch = pytest.importorskip("torch")
    ac = BytesAhoCorasick([b"ab"])
    offs = torch.zeros(3, dtype=torch.int64)
    for sb in (ac.is_match_stream_batch(2), ac.find_first_stream_batch(2), ac.count_matches_stream_batch(2, overlapping=True)):
        with pytest.raises(TypeError, match="uint8 CUDA tensor"):
            sb.feed_device(torch.zeros(4, dtype=torch.uint8), offs)   # a CPU tensor
        with pytest.raises(TypeError, match="uint8 CUDA tensor"):
            sb.feed_device(b"abcd", offs)
        assert sb.device is None


def test_single_query_stream_chunk_types_and_feed_after_finish():
    for make in ("is_match_stream", "find_first_stream", "count_matches_stream"):
        s = getattr(AhoCorasick(["ab"]), make)()
        with pytest.raises(TypeError, match="'str' expected"):
            s.feed(b"ab")
        b = getattr(BytesAhoCorasick([b"ab"]), make)()
        with pytest.raises(TypeError, match="not 'str'"):
            b.feed("ab")
        with pytest.raises(TypeError, match="contiguous"):
            b.feed(memoryview(b"abcdef")[::2])
        b._done = True   # what finish() leaves
        with pytest.raises(RuntimeError, match="feed after finish"):
            b.feed(b"ab")
