"""CPU tests of the stream search: the Python model of the device design (tests/stream_model.py) equals the oracle on the
concatenation after the last chunk, and the release rule's prefix after every chunk, on thousands of seeded cases; the
two C entry points refuse bad arguments before any CUDA call; the public objects validate their arguments before any
device work."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .stream_model import KIND_NAMES, ModelStream, released_by

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
SEARCHES = [(0, False), (1, False), (2, False), (0, True)]
SEARCH_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest", "Overlapping"]


def run_model(pats, kind, overlapping, chunks, over=None):
    """Feeds `chunks` to the model, checking the release rule after each; -> the rows released over all feeds."""
    full = Oracle(pats, KIND_NAMES[kind]).find(b"".join(chunks), overlapping=overlapping)
    st = ModelStream(pats, kind, overlapping, over)
    got, fed = [], 0
    for i, c in enumerate(chunks):
        last = i == len(chunks) - 1
        got += st.feed(c, last)
        fed += len(c)
        assert got == released_by(full, fed, kind, overlapping, st.max_len, last), (pats, chunks, i)
    assert got == full
    assert (st.fed, st.restart, st.tail) == (0, 0, b"")
    return got


def random_cuts(rng, n, max_len):
    """Cut points in [0, n]: lengths 0, 1, below, at and above max_pattern_len - 1, and long ones."""
    cuts, at = [], 0
    while at < n:
        r = rng.random()
        step = 0 if r < 0.1 else 1 if r < 0.25 else max(max_len - 1, 0) + int(rng.integers(-1, 2)) if r < 0.6 else int(rng.integers(1, 3 * max_len + 8))
        at = min(n, at + max(step, 0))
        cuts.append(at)
    return cuts


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_model_equals_the_oracle_on_seeded_cases(search):
    kind, overlapping = search
    rng = np.random.default_rng(7 + kind + 10 * overlapping)
    for case in range(900):
        shortest = 1 + case % 6
        pats = sorted({bytes(rng.integers(97, 100, size=int(rng.integers(shortest, shortest + 5))).astype(np.uint8)) for _ in range(12)})
        pats += pats[:1]   # a duplicate: distinct ids, same bytes
        hay = bytearray(rng.integers(97, 100, size=int(rng.integers(0, 120))).astype(np.uint8).tobytes())
        for _ in range(3):
            at = int(rng.integers(0, len(hay) + 1))
            hay[at:at] = pats[int(rng.integers(0, len(pats)))]
        hay = bytes(hay)
        cuts = random_cuts(rng, len(hay), max(len(p) for p in pats))
        chunks = [hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])]
        run_model(pats, kind, overlapping, chunks)


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
def test_cuts_at_every_offset_inside_planted_patterns(search):
    kind, overlapping = search
    pats = [b"abcd", b"bc", b"cdxyz", b"x", b"zab"]
    hay = b"qqabcdxyzabcdqq"
    for a in range(len(hay) + 1):
        for b in range(a, len(hay) + 1):
            run_model(pats, kind, overlapping, [hay[:a], hay[a:b], hay[b:]])


@pytest.mark.parametrize("search", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("pats", [[b"a", b"aa", b"aaa"], [b"a", b"b"], [b"aba", b"ab", b"ba", b"aba"]], ids=["nested", "single-byte", "self-overlap"])
def test_nested_self_overlapping_and_one_byte_patterns(search, pats):
    kind, overlapping = search
    rng = np.random.default_rng(len(pats))
    for _ in range(200):
        hay = rng.integers(97, 99, size=int(rng.integers(0, 40))).astype(np.uint8).tobytes()
        cuts = sorted(int(x) for x in rng.integers(0, len(hay) + 1, size=int(rng.integers(0, 8))))
        run_model(pats, kind, overlapping, [hay[a:b] for a, b in zip([0] + cuts, cuts + [len(hay)])])


def test_issue_example_leftmost_longest():
    """Patterns abcd, bc, LeftmostLongest: "xab" releases nothing; "cd" (5 bytes fed) releases (0, 1, 5)."""
    st = ModelStream([b"abcd", b"bc"], 2, False)
    assert st.feed(b"xab") == []
    assert st.feed(b"cd") == [(0, 1, 5)]
    assert st.feed(b"", True) == []


# ---------------------------------------------------------------- C entry points
def _automaton(kind=0, pats=(b"hello", b"world")):
    L = _capi.lib()
    offs = np.zeros(len(pats) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pats], out=offs[1:])
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pats), kind, -1, C.byref(h)) == 0
    return L, h


def _seams(L, h, data=FAKE, offs=FAKE, n=1, total=16, carry=FAKE, tail=FAKE, seam=FAKE, seam_offs=FAKE):
    return L.acb_stream_seams(h, data, offs, n, total, carry, tail, seam, seam_offs, None)


def _resolve(L, h, image=FAKE, data=FAKE, offs=FAKE, n=1, total=16, last=None, overlapping=0, codepoints=0, **ptrs):
    names = ["carry", "tail", "seam", "seam_offs", "seam_list", "seam_mo", "chunk_list", "chunk_mo", "scratch", "rows", "row_offs"]
    args = [ptrs.get(k, FAKE) for k in names]
    return L.acb_stream_resolve(h, image, data, offs, n, total, last, overlapping, codepoints, *args, None)


def test_entry_points_reject_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        seam_cases = [(dict(offs=None), "null argument"), (dict(carry=None), "null argument"), (dict(seam_offs=None), "null argument"),
                      (dict(data=None), "null argument"), (dict(tail=None), "null argument"), (dict(seam=None), "null argument"),
                      (dict(n=-1), "n_streams out of range"), (dict(n=0xffffffff), "n_streams out of range"),
                      (dict(total=1 << 31), "total_bytes must be below 2^31")]
        for kw, msg in seam_cases:
            assert _seams(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_stream_seams(None, FAKE, FAKE, 1, 16, FAKE, FAKE, FAKE, FAKE, None) == _capi.ACB_EINVAL
        names = ["carry", "tail", "seam", "seam_offs", "seam_list", "seam_mo", "chunk_list", "chunk_mo", "scratch", "rows", "row_offs"]
        resolve_cases = [({k: None}, "null argument") for k in names] + [
            (dict(offs=None), "null argument"), (dict(data=None), "null argument"),
            (dict(overlapping=2), "overlapping must be 0 or 1"), (dict(overlapping=-1), "overlapping must be 0 or 1"),
            (dict(codepoints=1, image=None), "code points need the device image"),
            (dict(n=-1), "n_streams out of range"), (dict(n=0xffffffff), "n_streams out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31")]
        for kw, msg in resolve_cases:
            assert _resolve(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


def test_one_byte_patterns_need_no_tail_or_seam_buffers():
    """max_pattern_len == 1: no tail, no seam.  Null buffers for them pass the null checks (the call then stops at the
    next check, the stream count)."""
    L, h = _automaton(0, (b"a", b"b"))
    try:
        assert _seams(L, h, tail=None, seam=None, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
        assert _resolve(L, h, tail=None, seam=None, n=-1) == _capi.ACB_EINVAL
        assert "n_streams out of range" in _capi.last_error()
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2])
def test_resolve_refuses_overlapping_on_a_leftmost_automaton(kind):
    L, h = _automaton(kind)
    try:
        assert _resolve(L, h, overlapping=1) == _capi.ACB_EUNSUPPORTED
        assert f"match kind {KIND_NAMES[kind]} does not support overlapping searches" in _capi.last_error()
        assert _resolve(L, h, overlapping=1, scratch=None) == _capi.ACB_EINVAL
    finally:
        L.acb_free(h)


# ---------------------------------------------------------------- Python validation (no device needed)
@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_overlapping_on_a_leftmost_automaton_is_refused_at_creation(kind):
    msg = f"match kind {kind.name} does not support overlapping searches"
    for ac in (AhoCorasick(["ab"], kind), BytesAhoCorasick([b"ab"], kind)):
        with pytest.raises(ValueError, match=msg):
            ac.stream(overlapping=True)
        with pytest.raises(ValueError, match=msg):
            ac.stream_batch(4, overlapping=True)


def test_a_batch_whose_seams_exceed_window_bytes_is_refused():
    """The seams of one feed (up to 2 x (max_pattern_len - 1) bytes per stream) are scanned in one call: a batch whose
    seams could exceed WINDOW_BYTES is refused when it is created, before any device work."""
    ac = BytesAhoCorasick([b"a" * 1025])
    limit = ac._ac.WINDOW_BYTES
    fits = limit // (2 * 1024)
    sb = ac.stream_batch(fits)
    assert sb.n_streams == fits and sb.device is None
    with pytest.raises(ValueError, match="seam bytes"):
        ac.stream_batch(fits + 1)
    with pytest.raises(ValueError, match="WINDOW_BYTES"):
        AhoCorasick(["é" * 5000]).stream_batch(1 << 20)


def test_stream_batch_argument_types():
    ac = BytesAhoCorasick([b"ab"])
    for bad in ("4", 4.0, True, None):
        with pytest.raises(TypeError):
            ac.stream_batch(bad)
    with pytest.raises(ValueError):
        ac.stream_batch(-1)
    sb = ac.stream_batch(2)
    torch = pytest.importorskip("torch")
    offs = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(torch.zeros(4, dtype=torch.uint8), offs)   # a CPU tensor
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(np.zeros(4, dtype=np.uint8), offs)
    with pytest.raises(TypeError, match="uint8 CUDA tensor"):
        sb.feed_device(b"abcd", offs)


def test_single_stream_chunk_types_and_feed_after_finish():
    s = AhoCorasick(["ab"]).stream()
    with pytest.raises(TypeError, match="'str' expected"):
        s.feed(b"ab")
    b = BytesAhoCorasick([b"ab"]).stream()
    with pytest.raises(TypeError, match="not 'str'"):
        b.feed("ab")
    with pytest.raises(TypeError):
        b.feed(12)
    with pytest.raises(TypeError, match="contiguous"):
        b.feed(memoryview(b"abcdef")[::2])
    b._done = True   # what finish() leaves
    with pytest.raises(RuntimeError, match="feed after finish"):
        b.feed(b"ab")


class _Huge:
    """A chunk that reports a length above one feed's limit without holding the bytes."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


def test_a_feed_above_window_bytes_is_refused_before_any_device_work():
    ac = BytesAhoCorasick([b"ab"])
    limit = ac._ac.WINDOW_BYTES
    s = ac.stream()
    with pytest.raises(ValueError, match="at most .* bytes"):
        s._feed(_Huge(limit + 1), False)
    assert s._offs is None and s._batch.device is None   # nothing was allocated on a device
    torch = pytest.importorskip("torch")

    class _Meta:   # a uint8 "CUDA tensor" of limit + 1 elements, without memory: only its metadata is read
        dtype, device = torch.uint8, torch.device("cuda", 0)

        def dim(self):
            return 1

        def numel(self):
            return limit + 1

    sb = ac.stream_batch(1)
    orig = torch.is_tensor
    torch.is_tensor = lambda x: isinstance(x, _Meta) or orig(x)
    try:
        offs = _Meta()
        offs.dtype, offs.shape = torch.int64, (2,)
        with pytest.raises(ValueError, match="WINDOW_BYTES"):
            sb.feed_device(_Meta(), offs)
    finally:
        torch.is_tensor = orig
    assert sb.device is None
