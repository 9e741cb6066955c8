"""Seeded inputs that steer the sieve (csrc/sieve.h, scan_sieve.cuh) into chosen corners of its geometry: reverse-trie
nodes with a given number of children, planted occurrences at chosen places of the 512-byte window grid, sparse
survivors a given number of windows apart, a window with more survivors than the first queue holds, and the dense
pattern shape that saturates a small filter.  Shared by the CPU interpreter tests and the GPU tests."""
from __future__ import annotations

import numpy as np

FANOUTS = (1, 8, 9, 255, 256)   # children of one trie node: linear scan (<= 8), binary search (> 8), the 9-bit count
TWO_LEVEL = "2x"                # a node with many children, each of which has many children again


def _csr(chunks):
    offs = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=offs[1:])
    data = np.frombuffer(b"".join(chunks) or b"\0", dtype=np.uint8)[: offs[-1]].copy()
    return data, offs


def _text(rng, nbytes, units):
    """Exactly nbytes bytes of random whole units (byte strings; one-byte units must be among them)."""
    ones = [u for u in units if len(u) == 1]
    pick = rng.integers(0, len(units), size=nbytes)
    alt = rng.integers(0, len(ones), size=nbytes)
    out, n, i = [], 0, 0
    while n < nbytes:
        u = units[pick[i]]
        if len(u) > nbytes - n:
            u = ones[alt[i]]
        out.append(u)
        n += len(u)
        i += 1
    return b"".join(out)


def _units(chars):
    return [c.encode() for c in chars]


PLANT_OFFSETS = (0, 1, 7, 8, 15, 16, 17, 495, 511)   # places in the 512-byte window grid (with the buffer 512-aligned)
HAY_LENGTHS = (0, 1, 15, 16, 17, 511, 512, 513, 16383, 16384, 16385)
GRID_HAY_BYTES = 40 * 1024 + 123
PAT_LENGTHS = (8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 23, 24, 29, 31, 32, 33, 37, 40)   # 16, 17: kSieveMaxLevel, + 1
LONG_PATTERN = 600                                      # longer than a window of text


class _Stream:
    """Haystacks built piece by piece; `pos` is the stream offset of the next byte."""

    def __init__(self, rng, filler):
        self.rng, self.filler = rng, filler
        self.hays, self.cur, self.pos = [], [], 0

    def put(self, b):
        self.cur.append(b)
        self.pos += len(b)

    def fill(self, n):
        self.put(_text(self.rng, n, self.filler))

    def fill_to(self, p):
        self.fill(p - self.pos)

    def end(self):
        self.hays.append(b"".join(self.cur))
        self.cur = []


def near_miss(p: bytes, which: int) -> bytes:
    """p with one one-byte character changed (the first, the last or a middle one, by `which`): no longer p."""
    s = p.decode("utf-8", "surrogateescape")
    idx = [i for i, c in enumerate(s) if c.isascii()]
    i = idx[[0, -1, len(idx) // 2][which % 3]]
    return (s[:i] + "#" + s[i + 1:]).encode("utf-8", "surrogateescape")


def planted_case(utf8: bool, seed: int = 0, decoys: int = 0):
    """-> (patterns, data, offsets) of the planted-occurrence batch.

    Patterns of 8..40 bytes (uppercase; with utf8 also 2- to 4-byte characters inside them), one of 600 bytes, suffixes
    and a prefix of another, duplicates, and QQQQQQQQ / QQQQQQQQQQQ.  The filler avoids their bytes (lowercase, space and,
    without utf8, raw bytes >= 0x80; with utf8, lowercase and 2- to 4-byte characters), so the survivors of the filter
    are mostly the planted ones.  Haystacks: the lengths of HAY_LENGTHS (each starting and, room permitting, ending with
    an occurrence; 16 and 17 are whole patterns), one of GRID_HAY_BYTES with an occurrence or a near miss per window,
    starting or ending at the PLANT_OFFSETS of the window grid, a sparse one (from a 16 KiB boundary of the stream)
    whose occurrences lie k windows apart for every k in 1..17 (twice), one with a run of 700 Q (a window with more
    survivors than the first queue holds), an occurrence cut by a haystack boundary, the long pattern and a near miss of
    it.  `decoys`: that many more patterns of 8..12 characters (digits; with utf8 also Greek letters) that the text
    never holds -- they fill the filters, not the match lists."""
    rng = np.random.default_rng(4242 + seed + (1 if utf8 else 0))
    pat_units = _units("ABCDEFGHIJKLMNOPRSTUVWXYZ") + (_units("ÉЖ€𝄞") if utf8 else [])
    filler = _units("abcdefghijklmnopqrstuvwxyz ") + (_units("éж€😀") if utf8 else [bytes([b]) for b in range(0x80, 0x100, 3)])
    pats = [_text(rng, n, pat_units) for n in PAT_LENGTHS]
    p24 = pats[PAT_LENGTHS.index(24)].decode()
    pats += [p24[-9:].encode(), p24[-12:].encode(), p24[:10].encode(), p24[3:14].encode()]   # nested, suffix-sharing
    pats += [b"Q" * 8, b"Q" * 11, pats[PAT_LENGTHS.index(16)], b"Q" * 8]                      # duplicates
    long = _text(rng, LONG_PATTERN, pat_units)
    pats.append(long)
    if decoys:
        dec_units = _units("0123456789") + (_units("αβγδεζηθ") if utf8 else [])
        dec = {_text(rng, int(rng.integers(8, 13)), dec_units) for _ in range(decoys)}
        pats += sorted(dec)
    short = pats[:len(PAT_LENGTHS) + 4]   # what is planted: the 8..40-byte patterns and the nested ones
    s = _Stream(rng, filler)
    k = 0

    def nxt():
        nonlocal k
        k += 1
        return short[(k * 7) % len(short)]

    for L in HAY_LENGTHS:
        if L in (16, 17):
            s.put(pats[PAT_LENGTHS.index(L)])
        elif L:
            a = nxt() if L >= 8 else b""
            a = a if len(a) <= L else b""
            s.put(a)
            b = nxt()
            if L - len(a) >= len(b) + 1:
                s.fill(L - len(a) - len(b))
                s.put(b)
            else:
                s.fill(L - len(a))
        s.end()
    # the grid haystack: one piece per window, starting (even modes) or ending (odd) at a place of the window grid
    start, w = s.pos, 0
    while True:
        base = ((s.pos >> 9) + 1) << 9
        o = PLANT_OFFSETS[w % len(PLANT_OFFSETS)]
        mode = (w // len(PLANT_OFFSETS)) % 4
        p = nxt()
        piece = p if mode < 2 else near_miss(p, w)
        at = base + o if mode % 2 == 0 else base + o - len(piece) + 1
        w += 1
        if at + len(piece) > start + GRID_HAY_BYTES:
            break
        if at < s.pos:
            continue
        s.fill_to(at)
        s.put(piece)
    s.fill_to(start + GRID_HAY_BYTES)
    s.end()
    # the sparse haystack, from the next 16 KiB boundary on (the task grid when the buffer is aligned)
    s.fill_to(((s.pos >> 14) + 1) << 14)
    s.end()
    win = (s.pos >> 9) + 2
    for rnd in range(2):
        for gap in range(1, 18):
            p = nxt()
            off = int(rng.integers(0, 512 - len(p) + 1)) if gap % 3 else int(rng.integers(0, 8))   # some reach into the history
            s.fill_to((win << 9) + off)
            s.put(p)
            win += gap
    s.fill_to((win + 1) << 9)
    s.end()
    # a run of Q: every position of a window survives the first probe
    s.fill(300)
    s.put(b"Q" * 700)
    s.fill(300)
    s.end()
    # an occurrence cut by a haystack boundary, then one at a haystack's start
    p31 = pats[PAT_LENGTHS.index(31)].decode()
    s.fill(100)
    s.put(p31[:15].encode())
    s.end()
    s.put(p31[15:].encode())
    s.fill(50)
    s.end()
    s.put(p31.encode())
    s.fill(40)
    s.end()
    # the long pattern, whole and with one byte changed
    s.fill(200)
    s.put(long)
    s.fill(300)
    s.put(near_miss(long, 2))
    s.fill(100)
    s.end()
    return pats, *_csr(s.hays)


def dense_case(utf8: bool, n_bytes: int = 1 << 20):
    """-> (patterns, data, offsets): the config-4 pattern shape (100 000 patterns of 5..8 lowercase letters) over
    n_bytes of lowercase text in 16 haystacks; with utf8 a 2- to 4-byte character every 37 bytes or so."""
    from ahocorasick_rs_b200 import workloads
    pats = workloads.random_lowercase_patterns(100_000, 5, 8, 4)
    rng = np.random.default_rng(44)
    if utf8:
        wide = _units("éж€😀")
        chunks, n = [], 0
        while n < n_bytes:
            c = rng.integers(97, 123, size=int(rng.integers(20, 55)), dtype=np.uint8).astype(np.uint8).tobytes() + wide[n % 4]
            chunks.append(c)
            n += len(c)
        text = b"".join(chunks)
        cuts = [0] + sorted(int(x) for x in rng.integers(0, len(text), size=15)) + [len(text)]
        # haystack boundaries at character starts
        cuts = [c if c == len(text) else next(i for i in range(c, len(text) + 1) if i == len(text) or text[i] & 0xC0 != 0x80)
                for c in cuts]
        hays = [text[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    else:
        text = rng.integers(97, 123, size=n_bytes, dtype=np.uint8).astype(np.uint8).tobytes()
        cuts = [0] + sorted(int(x) for x in rng.integers(0, n_bytes, size=15)) + [n_bytes]
        hays = [text[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    return pats, *_csr(hays)


def _child_bytes(rng, f):
    """f distinct preceding bytes, 0x00 and 0xff among them where f allows."""
    if f >= 256:
        return list(range(256))
    ends = [0x00, 0xFF][:f]
    rest = [b for b in rng.permutation(np.arange(1, 255)).tolist()][: f - len(ends)]
    return sorted(ends + rest)


def fanout_case(f, seed=0):
    """-> (patterns, data, offsets).  One 8-byte core; f patterns `b + core` (f = TWO_LEVEL: `b1 b2 + core` over 12 x
    10 pairs), plus the core itself (the node with the children is terminal too).  The text holds the core preceded by
    each of the 256 byte values (for TWO_LEVEL: every b2 after a listed b1, and every b1 before a listed b2), so it has
    the hits, the misses between children and the misses below the first and above the last child."""
    rng = np.random.default_rng(1000 + (257 if f == TWO_LEVEL else f) + 7919 * seed)
    core = bytes(rng.integers(0, 256, size=8, dtype=np.uint8).astype(np.uint8).tolist())
    sep = b"\x5c\x5c"
    if f == TWO_LEVEL:
        b2s, b1s = _child_bytes(rng, 12), _child_bytes(rng, 10)
        pats = [core] + [bytes([b1, b2]) + core for b2 in b2s for b1 in b1s]
        pieces = [bytes([b1s[i % len(b1s)], b2]) + core for i, b2 in enumerate(range(256))]
        pieces += [bytes([b1, b2s[i % len(b2s)]]) + core for i, b1 in enumerate(range(256))]
    else:
        pats = [core] + [bytes([b]) + core for b in _child_bytes(rng, f)]
        pieces = [bytes([b]) + core for b in range(256)]
    order = rng.permutation(len(pieces))
    hays, cur = [], b""
    for i, k in enumerate(order.tolist()):
        cur += pieces[k] + sep
        if i % 97 == 96:
            hays.append(cur)
            cur = b""
    hays.append(cur + core)   # the core alone, ending the last haystack
    return pats, *_csr(hays)
