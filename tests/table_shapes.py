"""Pattern sets aimed at each dense-table shape the builder makes (csrc/automaton.cpp step 4: range or class columns,
and ascii_rows_for: whether the byte-indexed table exists), with the shape each one must get, and the haystacks that
exercise them.  Shared by the CPU test (the image interpreter) and the GPU test (every kernel variant).

Each set covers its byte alphabet with patterns that no earlier pattern is a proper prefix of, so LeftmostFirst,
which drops such patterns before their bytes are counted as used, gives every match kind the same shape.  Sets with a
`lattice` pair (c0, c1) also hold the pattern c0 + c1 * 64, and c1 is in no other pattern: a run of c1 after any byte
is then quiet unless that byte is c0, and a byte that the walker confuses with c0 carries a false partial match across
the 64-byte chunk boundary."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from ahocorasick_rs_b200 import _capi

from . import image_interp as ii

RANGE, CLASS = 0, 1
LATTICE_BYTES = (0x7E, 0x7F, 0x80, 0xBF, 0xC0, 0xFF)   # the byte-indexed table's edge and the bytes it folds
LATTICE_RUN = 64


@dataclass
class Case:
    name: str
    pats: list
    mode: int
    n_cols: int
    col_lo: int
    byte_table: bool              # ascii_rows_for gives rows (every byte >= 0x7f is in the "other" column)
    alphabet: bytes
    lattice: tuple = None         # (c0, c1), see the module docstring
    colmap: dict = field(default_factory=dict)   # byte -> column the image must hold

    @property
    def wide(self):
        return self.n_cols == 256

    @property
    def outside(self):
        """Range columns: the bytes outside [lo, hi], which share the last column."""
        if self.mode != RANGE:
            return b""
        return bytes(b for b in range(256) if not self.col_lo <= b <= max(self.alphabet))


def _cover(alphabet, rng):
    """3-byte patterns that together use every byte of `alphabet`; equal lengths, so none is a prefix of another."""
    a = list(alphabet)
    rng.shuffle(a)
    while len(a) % 3:
        a.append(a[len(a) % len(alphabet)])
    return [bytes(a[i:i + 3]) for i in range(0, len(a), 3)]


def _extra(alphabet, n, lo, hi, rng):
    al = np.frombuffer(bytes(alphabet), dtype=np.uint8)
    return [bytes(al[rng.integers(0, len(al), size=int(rng.integers(lo, hi + 1)))]) for _ in range(n)]


def _case(name, alphabet, mode, n_cols, col_lo, byte_table, lattice=None, n_extra=40, lo=1, hi=4, colmap=None, seed=0):
    rng = np.random.default_rng(1000 + seed)
    alphabet = bytes(sorted(set(alphabet)))
    pats = []
    rest = alphabet
    if lattice:
        c0, c1 = lattice
        pats.append(bytes([c0]) + bytes([c1]) * LATTICE_RUN)
        rest = bytes(b for b in alphabet if b != c1)
    pats += _cover(rest, rng)
    # patterns that start with the highest byte, which is not a pattern by itself: a byte outside the range read
    # as the highest one starts a false partial match instead of trapping
    top = bytes([max(rest)])
    pats += [top + p for p in _extra(rest, 4, 1, 3, rng)]
    pats += [p for p in _extra(rest, n_extra, lo, hi, rng) if p != top]
    return Case(name, pats, mode, n_cols, col_lo, byte_table, alphabet, lattice, colmap or {})


def _bytes(lo, hi, skip=()):
    return bytes(b for b in range(lo, hi + 1) if b not in skip)


def _cases():
    out = [Case("one-byte", [b"a", b"aa", b"aaa", b"aaaaa"], RANGE, 2, 0x61, True, b"a",
                colmap={0x61: 0, 0x60: 1, 0x00: 1, 0x62: 1, 0x7F: 1, 0xFF: 1})]
    out.append(_case("lo-zero", _bytes(0x00, 0x05), RANGE, 7, 0x00, True, lattice=(0x05, 0x03), seed=1,
                     colmap={0x00: 0, 0x05: 5, 0x06: 6, 0x7F: 6, 0xFF: 6}))
    out.append(_case("hi-ff", _bytes(0xFA, 0xFF), RANGE, 7, 0xFA, False, seed=2,
                     colmap={0xFA: 0, 0xFF: 5, 0xF9: 6, 0x00: 6, 0x7F: 6}))
    gap = range(0x40, 0x70)
    out.append(_case("range-256", _bytes(0x00, 0xFE, gap), RANGE, 256, 0x00, False, n_extra=260, lo=2, hi=6, seed=3,
                     colmap={0x00: 0, 0x40: 0x40, 0xFE: 0xFE, 0xFF: 255}))
    gap = range(0x90, 0xC0)
    out.append(_case("range-from-1", _bytes(0x01, 0xFF, gap), RANGE, 256, 0x01, False, n_extra=260, lo=2, hi=6, seed=4,
                     colmap={0x01: 0, 0xFF: 254, 0x00: 255, 0x90: 0x8F}))
    out.append(_case("rule-5/4-range", b"abce", RANGE, 6, 0x61, True, seed=5, colmap={0x64: 3, 0x65: 4, 0x66: 5}))
    out.append(_case("rule-5/4-class", b"abcf", CLASS, 5, 0x61, True, seed=6,
                     colmap={0x61: 1, 0x63: 3, 0x64: 0, 0x66: 4, 0x67: 0}))
    out.append(_case("255-bytes", _bytes(0x00, 0xFF, (0x41,)), CLASS, 256, 0x00, False, n_extra=260, lo=2, hi=6, seed=7,
                     colmap={0x41: 0, 0x00: 1, 0x40: 0x41, 0x42: 0x42, 0xFF: 0xFF}))
    out.append(_case("256-bytes", _bytes(0x00, 0xFF), CLASS, 256, 0x00, False, n_extra=260, lo=2, hi=6, seed=8,
                     colmap={b: b for b in (0x00, 0x41, 0x7F, 0x80, 0xFF)}))
    out.append(_case("byte-table-range", _bytes(0x60, 0x7E), RANGE, 32, 0x60, True, lattice=(0x7E, 0x71), seed=9,
                     colmap={0x60: 0, 0x7E: 30, 0x7F: 31, 0x5F: 31, 0x80: 31}))
    out.append(_case("byte-table-class", b"acegikmoqsuwy~", CLASS, 15, 0x61, True, lattice=(0x7E, 0x71), seed=10,
                     colmap={0x61: 1, 0x7E: 14, 0x62: 0, 0x7F: 0, 0xFF: 0}))
    out.append(_case("no-byte-table-7f", _bytes(0x60, 0x7F), RANGE, 33, 0x60, False, lattice=(0x7F, 0x71), seed=11,
                     colmap={0x7E: 30, 0x7F: 31, 0x80: 32, 0x5F: 32}))
    return out


CASES = _cases()
CASE_IDS = [c.name for c in CASES]
WIDE = [c for c in CASES if c.wide]
BYTE_TABLE = [c for c in CASES if c.byte_table]
LATTICE = [c for c in CASES if c.lattice]
ASCII = [c for c in CASES if max(c.alphabet) < 0x80]   # patterns that are also str patterns


def hot_describe(im, max_rows):
    """acb_hot_bytes / acb_hot_build (no profile) / acb_hot_describe on the host -> HotDesc (rows, rows128, ...)."""
    L = im._L
    n = L.acb_hot_bytes(im._h, max_rows)
    buf = np.zeros(n, dtype=np.uint8)
    assert L.acb_hot_build(im._h, None, max_rows, buf.ctypes.data, n) == 0
    desc = _capi.HotDesc()
    assert L.acb_hot_describe(buf.ctypes.data, C.byref(desc)) == 0
    return desc


def check_shape(case, kind=0, max_rows=4096):
    """Assert the image and hot-image shape `case` was built for -> (Image, HotDesc)."""
    im = ii.Image(case.pats, kind)
    assert (im.col_mode, im.n_cols, im.col_lo) == (case.mode, case.n_cols, case.col_lo), case.name
    for b, col in case.colmap.items():
        assert im.colmap[b] == col, (case.name, hex(b))
        assert im.col(b) == col, (case.name, hex(b))
    if case.mode == CLASS and case.n_cols == 256 and len(case.alphabet) == 256:
        assert np.array_equal(im.colmap, np.arange(256)), "all 256 bytes used: the identity map"
    if case.mode == CLASS:   # every used byte has a column of its own, every other byte shares column 0
        used = np.zeros(256, dtype=bool)
        used[list(case.alphabet)] = True
        assert np.all((im.colmap != 0) == used) or len(case.alphabet) == 256
    desc = hot_describe(im, max_rows)
    assert desc.rows == min(max_rows, im.n_states - 1, 65535 // (2 * im.n_cols))
    assert (desc.rows128 > 0) == case.byte_table, case.name
    if case.byte_table:
        assert desc.rows128 == min(desc.rows, 255)
    return im, desc


# ---------------------------------------------------------------- haystacks
def plant(rng, arr, pats, n):
    """Write n patterns of `pats` over arr at random places (later ones may cut earlier ones)."""
    if len(arr) == 0:
        return arr
    for _ in range(n):
        p = pats[int(rng.integers(0, len(pats)))]
        if len(p) > len(arr):
            continue
        at = int(rng.integers(0, len(arr) - len(p) + 1))
        arr[at:at + len(p)] = np.frombuffer(p, dtype=np.uint8)
    return arr


def ragged_random(case, seed, n_haystacks=40, max_len=4000, empty=0.1):
    """A ragged batch of uniformly random bytes over 0x00-0xff with the case's patterns planted, and for range
    columns decoys: patterns that start with the highest byte, planted with a byte outside the range in its place
    -> (data, offsets)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, max_len + 1, size=n_haystacks)
    lens[rng.random(n_haystacks) < empty] = 0
    hays = []
    for n in lens:
        arr = rng.integers(0, 256, size=int(n), dtype=np.uint8).astype(np.uint8)
        plant(rng, arr, case.pats, int(n) // 24 + 1)
        if case.outside:
            top = max(case.alphabet)
            decoys = [bytes([case.outside[int(rng.integers(0, len(case.outside)))]]) + p[1:]
                      for p in case.pats if p[0] == top and len(p) > 1]
            plant(rng, arr, decoys, int(n) // 48 + 1)
        hays.append(arr)
    offs = np.zeros(n_haystacks + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    return np.concatenate(hays).astype(np.uint8) if hays else np.zeros(0, np.uint8), offs


def lattice_batch(case, seed):
    """Each of LATTICE_BYTES at every offset 0-63 of a 64-byte chunk (the data starts on the chunk grid).  Quiet
    blocks: c1 before and after the byte, so the only possible match is c0 + c1 * 64 (and only for the byte c0).  Busy
    blocks: random alphabet bytes, a pattern ending right before the byte and one starting right after it.  One
    haystack per lattice byte, 128-byte blocks -> (data, offsets)."""
    rng = np.random.default_rng(seed)
    c0, c1 = case.lattice
    others = case.pats[1:]
    al = np.frombuffer(bytes(b for b in case.alphabet if b != c1), dtype=np.uint8)
    hays = []
    for v in LATTICE_BYTES:
        blocks = []
        for k in range(64):
            q = np.full(128, c1, dtype=np.uint8)
            q[k] = v
            blocks.append(q)
            b = al[rng.integers(0, len(al), size=128)].copy()
            b[k] = v
            before, after = others[int(rng.integers(0, len(others)))], others[int(rng.integers(0, len(others)))]
            if len(before) <= k:
                b[k - len(before):k] = np.frombuffer(before, dtype=np.uint8)
            b[k + 1:k + 1 + len(after)] = np.frombuffer(after, dtype=np.uint8)
            blocks.append(b)
        hays.append(np.concatenate(blocks))
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return np.concatenate(hays), offs


UTF8_CHARS = ("é", "\u0080", "¿", "߿", "☃", "￯", "\U0001F926", "\U0010FFFF")


def utf8_texts(case, seed, n_random=30):
    """Code-point haystacks for an ASCII case -> list of str.  With a lattice, first: every character of UTF8_CHARS,
    and c0, followed by c1 * 64 with the character's last byte at every chunk offset it can reach (nb - 1 to 63 for
    an nb-byte character; each text is a multiple of 128 bytes, so in a
    batch that starts on the chunk grid they stay on it).  Then random mixes of the case's alphabet and 1- to 4-byte
    characters with its patterns planted."""
    rng = np.random.default_rng(seed)
    letters = [chr(b) for b in case.alphabet]
    pool = letters * 4 + list(UTF8_CHARS)
    texts = []
    if case.lattice:
        c0, c1 = (chr(x) for x in case.lattice)
        for ch in UTF8_CHARS + (c0,):
            nb = len(ch.encode())
            texts.append("".join(c1 * k + ch + c1 * (128 - k - nb) for k in range(0, 65 - nb)))
    for _ in range(n_random):
        n = int(rng.integers(0, 1500))
        parts = [pool[int(i)] for i in rng.integers(0, len(pool), size=n)]
        for _ in range(n // 20):
            at = int(rng.integers(0, len(parts) + 1))
            parts.insert(at, case.pats[int(rng.integers(0, len(case.pats)))].decode())
        texts.append("".join(parts))
    return texts


def batch_of(hays):
    """list of bytes -> (data, offsets)"""
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return np.frombuffer(b"".join(hays) or b"\0", dtype=np.uint8)[:offs[-1]].copy(), offs
