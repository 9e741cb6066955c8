"""CPU tests of the match-mask stream: the Python model of the device design (tests/stream_mask_model.py) releases, after
every feed, exactly the prefix [0, R) of the one-shot mask (the union of the oracle's record spans of the
concatenation), R = max(0, F - (max_pattern_len - 1)), and the whole mask at `last`; the two C entry points refuse bad
arguments before any CUDA call; the public objects validate their arguments before any device work."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi
from oracle import Oracle

from .stream_mask_model import KIND_NAMES, MaskModelStream, one_shot_mask, released_positions
from .test_stream_cpu import random_cuts

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
SEARCHES = [(0, False), (1, False), (2, False), (0, True)]
SEARCH_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest", "Overlapping"]


def run_model(pats, kind, overlapping, flows, st=None, admitted=None):
    """Feeds each flow (a list of chunks, the last one fed with `last`) to one model stream, the slot reused from flow to
    flow, checking the released prefix after every feed and the whole mask at `last`."""
    sub = pats if admitted is None else [p for i, p in enumerate(pats) if i in admitted]
    if st is None:
        st = MaskModelStream(pats, kind, overlapping, Oracle(sub, "Standard") if admitted is not None else None)
    for chunks in flows:
        hay = b"".join(chunks)
        full = one_shot_mask(sub, kind, overlapping, hay) if sub else [0] * len(hay)
        got, fed = [], 0
        for i, c in enumerate(chunks):
            last = i == len(chunks) - 1
            r_old, flags = st.feed(c, last)
            assert r_old == len(got), (pats, chunks, i)
            got += flags
            fed += len(c)
            r = fed if last else max(0, fed - st.halo)
            assert len(got) == r, (pats, chunks, i)
            assert got == full[:r], (pats, chunks, i)
        assert got == full
        assert st.rows.fed == 0 and st.held == []
    return st


def cut(hay, cuts):
    return [hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])]


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_model_equals_the_one_shot_mask_on_seeded_cases(search):
    kind, overlapping = search
    rng = np.random.default_rng(11 + kind + 10 * overlapping)
    for case in range(600):
        shortest = 1 + case % 6
        pats = sorted({bytes(rng.integers(97, 100, size=int(rng.integers(shortest, shortest + 5))).astype(np.uint8)) for _ in range(12)})
        pats += pats[:1]   # a duplicate: distinct ids, same bytes
        hay = bytearray(rng.integers(97, 100, size=int(rng.integers(0, 120))).astype(np.uint8).tobytes())
        for _ in range(3):
            at = int(rng.integers(0, len(hay) + 1))
            hay[at:at] = pats[int(rng.integers(0, len(pats)))]
        hay = bytes(hay)
        run_model(pats, kind, overlapping, [cut(hay, random_cuts(rng, len(hay), max(len(p) for p in pats)))])


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_cuts_at_every_offset_inside_planted_patterns(search):
    kind, overlapping = search
    pats = [b"abcd", b"bc", b"cdxyz", b"x", b"zab"]
    hay = b"qqabcdxyzabcdqq"
    st = None
    for a in range(len(hay) + 1):
        for b in range(a, len(hay) + 1):
            st = run_model(pats, kind, overlapping, [[hay[:a], hay[a:b], hay[b:]]], st)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("pats", [[b"a", b"aa", b"aaa"], [b"a", b"b"], [b"aba", b"ab", b"ba", b"aba"]], ids=["nested", "single-byte", "self-overlap"])
def test_nested_self_overlapping_and_one_byte_patterns(search, pats):
    """[a, b]: max_pattern_len 1, halo 0 -- every byte is released by the feed that brings it, nothing is held."""
    kind, overlapping = search
    rng = np.random.default_rng(len(pats))
    st = MaskModelStream(pats, kind, overlapping)
    for _ in range(200):
        hay = rng.integers(97, 99, size=int(rng.integers(0, 40))).astype(np.uint8).tobytes()
        cuts = sorted(int(x) for x in rng.integers(0, len(hay) + 1, size=int(rng.integers(0, 8))))
        run_model(pats, kind, overlapping, [cut(hay, cuts)], st)
        if st.halo == 0:
            assert st.held == []


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_chunks_shorter_and_longer_than_the_tail_and_empty_ones(search):
    """Long patterns (halo 40): chunks of 0, 1, halo - 1, halo, halo + 1 and 3 x halo bytes in every order."""
    kind, overlapping = search
    rng = np.random.default_rng(5 + kind)
    pats = [b"ab" * 20 + b"c", b"ba" * 5, b"abab", b"b" * 30, b"cab"]
    halo = max(len(p) for p in pats) - 1
    st = MaskModelStream(pats, kind, overlapping)
    for _ in range(60):
        lens = [int(x) for x in rng.choice([0, 1, halo - 1, halo, halo + 1, 3 * halo], size=int(rng.integers(1, 8)))]
        hay = bytes(rng.choice(np.frombuffer(b"abbc", dtype=np.uint8), size=sum(lens)).astype(np.uint8))
        hay = hay[:len(hay) // 2] + pats[0] + hay[len(hay) // 2:]
        cuts = list(np.cumsum(lens[:-1])) if len(lens) > 1 else []
        run_model(pats, kind, overlapping, [cut(hay, [min(int(c), len(hay)) for c in cuts])], st)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_a_slot_reused_after_last(search):
    """Three flows through one slot: each starts again at position 0 with no held flags left from the one before."""
    kind, overlapping = search
    pats = [b"hello", b"lo w", b"world", b"ow"]
    flows = [[b"say hel", b"lo w", b"orld"], [b"", b"world"], [b"lo", b" wo", b"rld!", b""]]
    st = run_model(pats, kind, overlapping, flows)
    run_model(pats, kind, overlapping, flows[::-1], st)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_admitted_subsets(search):
    """A stream that searches for a subset keeps the full automaton's tail (halo of the longest pattern of all), and
    its mask is the subset's one-shot mask; an unadmitted long pattern over an admitted short one hides nothing."""
    kind, overlapping = search
    rng = np.random.default_rng(23 + kind)
    pats = [b"abcabcab", b"bca", b"ca", b"cab", b"a", b"bcabc"]
    for case in range(150):
        admitted = {i for i in range(len(pats)) if rng.random() < 0.5}
        hay = bytes(rng.choice(np.frombuffer(b"abc", dtype=np.uint8), size=int(rng.integers(0, 60))).astype(np.uint8))
        run_model(pats, kind, overlapping, [cut(hay, random_cuts(rng, len(hay), 8))], admitted=admitted)


def _encode(ids):
    return bytes(b for t in ids for b in (0x80 | (t >> 14), (t >> 7) & 0x7F, t & 0x7F))


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_released_positions_per_feed_follow_the_rule_in_bytes_and_at_stride_3(search):
    """Token ids (3 bytes each): a feed releases ceil(R_new / 3) - ceil(R_old / 3) tokens, all but the last k - 1 fed
    (k the longest pattern in tokens) before `last`, and their flags are the per-token one-shot mask."""
    kind, overlapping = search
    rng = np.random.default_rng(31 + kind)
    tok_pats = [[5, 300], [300, 5, 300], [7], [300, 300, 70000, 5]]
    pats = [_encode(p) for p in tok_pats]
    k = max(len(p) for p in tok_pats)
    for _ in range(100):
        ids = [int(x) for x in rng.choice([5, 7, 300, 70000], size=int(rng.integers(0, 40)))]
        cuts = sorted(int(x) for x in rng.integers(0, len(ids) + 1, size=int(rng.integers(0, 6))))
        chunks = [_encode(ids[a:b]) for a, b in zip([0] + cuts, cuts + [len(ids)])]
        full = one_shot_mask(pats, kind, overlapping, b"".join(chunks))
        st = MaskModelStream(pats, kind, overlapping)
        got, tokens_fed = [], 0
        for i, c in enumerate(chunks):
            last = i == len(chunks) - 1
            r_old, flags = st.feed(c, last)
            fed = st.rows.fed if not last else len(full)
            r_new = r_old + len(flags)
            assert len(flags) == r_new - r_old and r_new == (fed if last else max(0, fed - (3 * k - 1)))
            first, tok_flags = released_positions(r_old, flags, 3)
            assert first == len(got) and len(tok_flags) == -(-r_new // 3) - -(-r_old // 3)
            tokens_fed += len(c) // 3
            assert first + len(tok_flags) == (tokens_fed if last else max(0, tokens_fed - (k - 1)))
            got += tok_flags
        assert got == full[::3]


# ---------------------------------------------------------------- C entry points
def _automaton(kind=0, pats=(b"hello", b"world")):
    L = _capi.lib()
    offs = np.zeros(len(pats) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pats], out=offs[1:])
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pats), kind, -1, C.byref(h)) == 0
    return L, h


ROWS_NAMES = ["offs", "carry", "seam_offs", "rows", "row_offs", "chunk_mask", "seam_mask"]
EMIT_NAMES = ["offs", "carry", "seam_offs", "chunk_mask", "seam_mask", "held_in", "held_out", "flags", "flag_offs", "flag_starts"]


def _rows(L, n=1, **ptrs):
    p = [ptrs.get(k, FAKE) for k in ROWS_NAMES]
    return L.acb_stream_mask_rows(p[0], n, *p[1:], None)


def _emit(L, h, n=1, last=None, overlapping=0, stride=1, **ptrs):
    p = {k: ptrs.get(k, FAKE + 64 * i) for i, k in enumerate(EMIT_NAMES)}
    return L.acb_stream_mask_emit(h, p["offs"], n, last, overlapping, stride, *[p[k] for k in EMIT_NAMES[1:]], None)


def test_entry_points_reject_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        rows_cases = [({k: None}, "null argument") for k in ROWS_NAMES] + [
            (dict(n=-1), "n_streams out of range"), (dict(n=0xffffffff), "n_streams out of range")]
        for kw, msg in rows_cases:
            assert _rows(L, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        emit_cases = [({k: None}, "null argument") for k in EMIT_NAMES] + [
            (dict(held_out=FAKE + 64 * EMIT_NAMES.index("held_in")), "different buffers"),
            (dict(overlapping=2), "overlapping must be 0 or 1"), (dict(overlapping=-1), "overlapping must be 0 or 1"),
            (dict(stride=0), "stride out of range"), (dict(stride=1 << 32), "stride out of range"),
            (dict(n=-1), "n_streams out of range"), (dict(n=0xffffffff), "n_streams out of range")]
        for kw, msg in emit_cases:
            assert _emit(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_stream_mask_emit(None, FAKE, 1, None, 0, 1, *[FAKE + 64 * i for i in range(9)], None) == _capi.ACB_EINVAL
        assert "null argument" in _capi.last_error()
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


def test_one_byte_patterns_need_no_held_flags():
    """max_pattern_len == 1: nothing is held.  Null (or equal) held buffers pass their checks; the call stops at the
    next check, the stream count."""
    L, h = _automaton(0, (b"a", b"b"))
    try:
        assert _emit(L, h, held_in=None, held_out=None, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
        assert _emit(L, h, held_in=FAKE, held_out=FAKE, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2])
def test_emit_refuses_overlapping_on_a_leftmost_automaton(kind):
    L, h = _automaton(kind)
    try:
        launches = L.acb_launch_count()
        assert _emit(L, h, overlapping=1) == _capi.ACB_EUNSUPPORTED
        assert f"match kind {KIND_NAMES[kind]} does not support overlapping searches" in _capi.last_error()
        assert _emit(L, h, overlapping=1, flags=None) == _capi.ACB_EINVAL   # argument errors come first
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


def test_the_new_entry_points_are_exported():
    L = _capi.lib()
    for name in ("acb_stream_mask_rows", "acb_stream_mask_emit"):
        assert name in _capi.EXPORTS
        getattr(L, name)


# ---------------------------------------------------------------- Python validation (no device needed)
@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_overlapping_on_a_leftmost_automaton_is_refused_at_creation(kind):
    msg = f"match kind {kind.name} does not support overlapping searches"
    for ac in (AhoCorasick(["ab"], kind), BytesAhoCorasick([b"ab"], kind), TokenAhoCorasick([[1, 2]], kind)):
        with pytest.raises(ValueError, match=msg):
            ac.match_mask_stream_batch(4, overlapping=True)
        with pytest.raises(ValueError, match=msg):
            ac.match_spans_stream(overlapping=True)


def test_too_many_streams_are_refused_at_creation():
    ac = BytesAhoCorasick([b"a" * 1025])
    fits = ac._ac.WINDOW_BYTES // (2 * 1024)
    sb = ac.match_mask_stream_batch(fits)
    assert sb.n_streams == fits and sb.device is None
    with pytest.raises(ValueError, match="seam bytes"):
        ac.match_mask_stream_batch(fits + 1)
    with pytest.raises(ValueError, match="WINDOW_BYTES"):
        AhoCorasick(["é" * 5000]).match_mask_stream_batch(1 << 20)
    with pytest.raises(ValueError, match="seam bytes"):
        TokenAhoCorasick([list(range(400))]).match_mask_stream_batch(1 << 20)


def test_batch_argument_types():
    ac = BytesAhoCorasick([b"ab"])
    for bad in ("4", 4.0, True, None):
        with pytest.raises(TypeError):
            ac.match_mask_stream_batch(bad)
    with pytest.raises(ValueError):
        ac.match_mask_stream_batch(-1)
    with pytest.raises(ValueError, match="give both or neither"):
        ac.match_mask_stream_batch(2, set_index=object())
    sb = ac.match_mask_stream_batch(2)
    torch = pytest.importorskip("torch")
    offs = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(torch.zeros(4, dtype=torch.uint8), offs)   # a CPU tensor
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(torch.zeros(4, dtype=torch.int32), offs)
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(np.zeros(4, dtype=np.uint8), offs)
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(b"abcd", offs)
    assert sb.device is None


def test_host_stream_chunk_types_and_feed_after_finish():
    s = AhoCorasick(["ab"]).match_spans_stream()
    with pytest.raises(TypeError, match="'str' expected"):
        s.feed(b"ab")
    b = BytesAhoCorasick([b"ab"]).match_spans_stream()
    with pytest.raises(TypeError, match="not 'str'"):
        b.feed("ab")
    with pytest.raises(TypeError):
        b.feed(12)
    with pytest.raises(TypeError, match="contiguous"):
        b.feed(memoryview(b"abcdef")[::2])
    t = TokenAhoCorasick([[1, 2]]).match_spans_stream()
    with pytest.raises(TypeError):
        t.feed(["a"])
    with pytest.raises(ValueError, match="outside"):
        t.feed([1 << 21])
    assert b.released == 0 and t.released == 0
    for st in (s, b, t):
        (st._stream if hasattr(st, "_stream") else st)._done = True   # what finish() leaves
    with pytest.raises(RuntimeError, match="feed after finish"):
        b.feed(b"ab")
    with pytest.raises(RuntimeError, match="feed after finish"):
        s.feed("ab")
    with pytest.raises(RuntimeError, match="feed after finish"):
        t.feed([1, 2])
