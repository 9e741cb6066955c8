"""GPU tests (-m gpu) of the staged walker's lazily built per-lane record and of its narrow warm-up fetch.

A lane keeps the exact scanner's state and its segment bookkeeping nowhere until it first needs the exact scanner;
they are then derived again from the task, the lane and what the fast path has done since (whether the warm-up has
ended, the guessed start state).  These inputs put that first hand-over at every place it can happen -- inside the
warm-up bytes, in the first and the last 16-byte group of a segment, at a haystack end in the middle of a segment --
and put leftmost matches across the warm-up end and the segment end, short haystacks behind a lane whose record was
built late, and segments outside the stream on both sides.  The warm-up bytes are fetched unit by unit from where
the warm-up starts, so warm-ups of 16, 64 and 128 bytes run with the buffer 1, 16 and 63 bytes off the copy grid.
Every staged variant (one / two segments per lane, compact / byte-indexed table), bytes and code points, the three
match kinds and the overlapping search, compared with the CPU oracle bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from .gpu_helpers import SEARCH_IDS, SEARCHES, check_batch, make_ac, set_kernel  # noqa: E402

S = 1024   # the default segment size; patterns of up to 128 bytes keep it (a segment is at least 8 warm-ups)
# name -> acb_set_tuning(kernel, hot_rows, segment_bytes, table)
STAGED = {
    "one-per-lane-compact": (2, 0, 0, 1),
    "one-per-lane-byte-table": (2, 0, 0, 2),
    "two-per-lane-compact": (3, 0, 0, 1),
    "two-per-lane-byte-table": (3, 0, 0, 2),
}
LONG = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789+/" * 2   # 128 bytes, no repeated letter within 64


@pytest.fixture(params=list(STAGED))
def staged(request):
    set_kernel(*STAGED[request.param])
    try:
        yield request.param
    finally:
        set_kernel(0)


def haystack(rng, n, plants, codepoints):
    """n bytes of filler that is part of no pattern, with `plants` [(position, bytes)] written over it; for code
    points some of the untouched filler becomes two-byte characters."""
    arr = rng.choice(np.frombuffer(b"#$%&*-=_ ", dtype=np.uint8), size=n)
    taken = np.zeros(n + 1, dtype=bool)
    taken[n] = True
    for pos, p in plants:
        assert 0 <= pos and pos + len(p) <= n, (pos, len(p), n)
        arr[pos:pos + len(p)] = np.frombuffer(p, dtype=np.uint8)
        taken[pos:pos + len(p)] = True
    if codepoints:
        for i in rng.integers(0, max(n - 1, 1), size=n // 6):
            if n >= 2 and not taken[i] and not taken[i + 1]:
                arr[i:i + 2] = (0xC3, 0xA9)   # é
                taken[i:i + 2] = True
    return arr


def assemble(lead, hays, tail):
    """-> (buffer, offsets): `lead` bytes before the stream and `tail` after it that belong to no haystack."""
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return np.concatenate([lead, *hays, tail]).astype(np.uint8), offs + len(lead)


def staged_stats(ac):
    st = ac._ac.last_stats
    assert st["engine"] == "table" and st["segment_bytes"] == S
    return st


@pytest.mark.parametrize("codepoints", [False, True], ids=["bytes", "codepoints"])
@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
def test_first_hand_over_everywhere(kind, overlapping, codepoints, staged):
    rng = np.random.default_rng(7)
    long16 = LONG[:16]
    pats = [long16, b"abc", b"ab", b"+"]   # the long one first: LeftmostFirst keeps "ab" pending while it can still win
    start = 2 * S + 40                     # of the stream inside the buffer: segments 0 and 1 lie before it

    def at(pos):                           # buffer position -> position in the first haystack
        return pos - start

    first = haystack(rng, 14 * S - 300 - start, [
        (at(4 * S - 7), b"ab"),            # ends inside segment 4's warm-up bytes, and in the last group of segment 3
        (at(5 * S + 2), b"+"),             # the first group of segment 5, whose lane has scanned nothing else yet
        (at(5 * S + 600), b"abc"),         # ... and then reports a second match from its head piece
        (at(6 * S - 8), long16),           # pending across segment 6's warm-up end and segment 5's end
        (at(8 * S - 6), long16[:12]),      # pending across the seam, then falls back to "abc" behind it
        (at(9 * S - 3), b"+"),             # the last group of segment 8
        (at(10 * S - 1), b"ab"),           # a match on the seam itself
        (at(12 * S - 16), long16),         # exactly the warm-up bytes
    ], codepoints)
    # the first haystack ends inside segment 13: that lane builds its record there and goes on through these
    short = [haystack(rng, n, [(p, b) for p, b in pl if p + len(b) <= n], codepoints)
             for n, pl in [(20, [(3, b"ab")]), (0, []), (35, [(30, b"abc")]), (1, []), (50, [(0, b"+"), (47, b"abc")])]]
    last = haystack(rng, S + 77, [(S - 40, long16), (S + 70, b"ab")], codepoints)
    lead = haystack(rng, start, [(100, b"ab"), (start - 2, b"ab")], False)   # not part of any haystack
    tail = haystack(rng, 3 * S + 5, [(0, b"bc"), (S, long16)], False)        # segments past the stream
    data, offs = assemble(lead, [first, *short, last], tail)
    ac = make_ac(pats, kind, codepoints)
    assert check_batch(pats, kind, data, offs, overlapping, codepoints, ac=ac) >= 14
    st = staged_stats(ac)
    assert st["traps"] >= 10 and st["segments"] >= 18


@pytest.mark.parametrize("shift", [1, 16, 63])
@pytest.mark.parametrize("warm", [16, 64, 128])
def test_warm_up_lengths_off_the_copy_grid(warm, shift, staged):
    """A pattern of `warm` bytes makes the warm-up that long.  Byte i of the data lies at grid position i + shift, so
    the warm-up starts in any of the four 16-byte units of its chunk and, for 64 and 128, spans two or three chunks."""
    long_p = LONG[:warm]
    pats = [long_p, long_p[:warm // 2], b"ab", b"+"]

    def seam(k, delta):   # data index of grid position k * S + delta
        return k * S - shift + delta

    for codepoints in (False, True):
        rng = np.random.default_rng(100 * warm + shift)
        first = haystack(rng, 9 * S + 123, [
            (seam(1, -warm // 2), long_p),          # half in the warm-up, half in the segment
            (seam(2, -1), long_p),                  # one byte before the seam
            (seam(3, 1 - warm), long_p),            # ends one byte into the segment
            (seam(4, -warm), long_p),               # exactly the warm-up bytes
            (seam(5, -warm + 3), long_p[:warm - 3] + b"#"),   # all but its end, across the seam: falls back to the half
            (seam(6, 0), b"+"),
            (seam(7, -1), b"+"),
            (seam(8, -warm - 1), b"ab"),            # just before the warm-up: the guess must not know of it
        ], codepoints)
        others = [haystack(rng, n, [(n // 2, b"ab")] if n > 4 else [], codepoints) for n in (70, 0, 3, 200)]
        last = haystack(rng, 3 * S, [(S - warm // 4, long_p), (3 * S - warm, long_p)], codepoints)
        data, offs = assemble(np.zeros(0, np.uint8), [first, *others, last], np.zeros(0, np.uint8))
        for kind, overlapping in SEARCHES:
            ac = make_ac(pats, kind, codepoints)
            assert check_batch(pats, kind, data, offs, overlapping, codepoints, ac=ac, shift=shift) >= 12
            st = staged_stats(ac)
            assert st["traps"] > 0
