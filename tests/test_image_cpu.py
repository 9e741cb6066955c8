"""CPU tests of the PRODUCT's host side and kernel logic: the automaton builder /
device image / hot image (csrc/automaton.cpp) and the control flow of the
kernels -- exact scanner, segment kernel with speculative starts, repair pass,
ordering and code point fix-up -- executed by the Python image interpreter
(tests/image_interp.py) and compared with the oracle.  No GPU needed; the GPU
parity tests proper are in test_gpu_parity.py."""
import json
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from oracle import Oracle
from tests import image_interp as ii
from tests.spec_bruteforce import spec_find

HERE = os.path.dirname(os.path.abspath(__file__))
KINDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]
KID = {"Standard": 0, "LeftmostFirst": 1, "LeftmostLongest": 2}

with open(os.path.join(HERE, "golden", "reference_vectors.json"), encoding="utf-8") as f:
    VECTORS = [v for v in json.load(f)["vectors"] if not v.get("error")]


def batch(hays):
    data = np.frombuffer(b"".join(hays) or b"\0", dtype=np.uint8)
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hays], out=offs[1:])
    return data, offs


def oracle_batch(orc, hays, overlapping=False, cp=False):
    out = []
    for h, hay in enumerate(hays):
        ms = orc.find_str(hay.decode(), overlapping) if cp else orc.find(hay, overlapping)
        out += [(h, p, s, e) for (p, s, e) in ms]
    return out


@pytest.mark.parametrize("vec", VECTORS, ids=[f"{i}:{v['src']}" for i, v in enumerate(VECTORS)])
def test_image_reproduces_reference_vectors(vec):
    pats = [p.encode("utf-8") for p in vec["patterns"]]
    im = ii.Image(pats, KID[vec["kind"]])
    hay = vec["haystack"]
    raw = hay.encode("utf-8")
    cp = vec["cls"] == "str"
    got = ii.find(im, raw, vec["overlapping"], cp)
    for H in (2, 3, 7, 40):
        for base in (0, 5, 64 - 3):
            assert ii.find_staged(im, raw, vec["overlapping"], cp, H=H, base_addr=base, segment_bytes=64) == got
    if "expect_strings" in vec:
        if cp:
            assert [hay[s:e] for (_, s, e) in got] == vec["expect_strings"]
        else:
            assert [raw[s:e].decode() for (_, s, e) in got] == vec["expect_strings"]
    if "expect_indexes" in vec:
        assert [list(m) for m in got] == vec["expect_indexes"]


def alpha(k, max_size, min_size=1):
    return st.binary(min_size=min_size, max_size=max_size).map(lambda b: bytes(97 + (x % k) for x in b))


@settings(max_examples=250, deadline=None)
@given(st.lists(alpha(2, 5), min_size=1, max_size=8), alpha(2, 700, 0), st.sampled_from(KINDS), st.integers(1, 30),
       st.integers(0, 63))
def test_segments_and_repair_match_oracle_ab(patterns, haystack, kind, H, base):
    """Dense matches on a two-letter alphabet with 128-byte segments: nearly every
    segment boundary needs the repair pass."""
    orc = Oracle(patterns, kind)
    im = ii.Image(patterns, KID[kind])
    exp = orc.find(haystack)
    assert ii.find(im, haystack) == exp
    assert ii.find_staged(im, haystack, H=H, base_addr=base, segment_bytes=128) == exp
    if kind == "Standard":
        expo = orc.find(haystack, overlapping=True)
        assert ii.find(im, haystack, overlapping=True) == expo
        assert ii.find_staged(im, haystack, overlapping=True, H=H, base_addr=base, segment_bytes=128) == expo


@settings(max_examples=150, deadline=None)
@given(st.lists(alpha(3, 6), min_size=1, max_size=12), alpha(3, 900, 0), st.sampled_from(KINDS), st.integers(1, 60),
       st.integers(0, 63))
def test_segments_and_repair_match_oracle_abc(patterns, haystack, kind, H, base):
    orc = Oracle(patterns, kind)
    im = ii.Image(patterns, KID[kind])
    exp = orc.find(haystack)
    assert exp == spec_find(patterns, haystack, kind) or len(haystack) > 300  # brute force only on the small ones
    assert ii.find_staged(im, haystack, H=H, base_addr=base, segment_bytes=128) == exp


@settings(max_examples=120, deadline=None)
@given(st.lists(alpha(2, 24, 1), min_size=1, max_size=5), alpha(2, 1500, 200), st.sampled_from(KINDS),
       st.integers(0, 63))
def test_long_patterns_across_boundaries(patterns, haystack, kind, base):
    """Patterns up to 24 bytes (warm-up of 32) and pending leftmost matches that straddle segment boundaries."""
    orc = Oracle(patterns, kind)
    im = ii.Image(patterns, KID[kind])
    assert ii.find_staged(im, haystack, base_addr=base, segment_bytes=64) == orc.find(haystack)


@settings(max_examples=120, deadline=None)
@given(st.lists(alpha(2, 4), min_size=1, max_size=6), st.lists(alpha(2, 400, 0), min_size=1, max_size=8),
       st.sampled_from(KINDS), st.integers(1, 20), st.integers(0, 63), st.integers(0, 40))
def test_ragged_batches(patterns, hays, kind, H, base, shift):
    """Several haystacks per segment, haystacks spanning segments, empty haystacks, offsets[0] > 0."""
    orc = Oracle(patterns, kind)
    im = ii.Image(patterns, KID[kind])
    data, offs = batch(hays)
    data = np.concatenate([np.full(shift, 98, dtype=np.uint8), data])
    offs = offs + shift
    exp = oracle_batch(orc, hays)
    assert ii.emulate_plain(im, data, offs) == exp
    assert ii.emulate_scan(im, data, offs, H=H, base_addr=base, segment_bytes=128) == exp
    if kind == "Standard":
        expo = oracle_batch(orc, hays, overlapping=True)
        assert ii.emulate_scan(im, data, offs, overlapping=True, H=H, base_addr=base, segment_bytes=128) == expo


@settings(max_examples=120, deadline=None)
@given(st.lists(st.binary(min_size=1, max_size=4), min_size=1, max_size=10), st.binary(max_size=300),
       st.sampled_from(KINDS), st.integers(1, 40))
def test_image_binary_patterns(patterns, haystack, kind, H):
    orc = Oracle(patterns, kind)
    im = ii.Image(patterns, KID[kind])
    exp = orc.find(haystack)
    assert ii.find(im, haystack) == exp
    assert ii.find_staged(im, haystack, H=H, segment_bytes=128) == exp


TEXT = "abé☃\U0001F926 "


@settings(max_examples=150, deadline=None)
@given(st.lists(st.text(alphabet="abé☃\U0001F926", min_size=1, max_size=3), min_size=1, max_size=6),
       st.lists(st.text(alphabet=TEXT, max_size=150), min_size=1, max_size=4), st.sampled_from(KINDS),
       st.integers(1, 30), st.integers(0, 63))
def test_code_points(patterns, hays, kind, H, base):
    pats = [p.encode() for p in patterns]
    orc = Oracle(pats, kind)
    im = ii.Image(pats, KID[kind])
    raws = [h.encode() for h in hays]
    data, offs = batch(raws)
    exp = oracle_batch(orc, raws, cp=True)
    assert ii.emulate_plain(im, data, offs, cp=True) == exp
    assert ii.emulate_scan(im, data, offs, cp=True, H=H, base_addr=base, segment_bytes=128) == exp
    if kind == "Standard":
        expo = oracle_batch(orc, raws, overlapping=True, cp=True)
        assert ii.emulate_scan(im, data, offs, overlapping=True, cp=True, H=H, base_addr=base, segment_bytes=128) == expo


def test_never_converging_repair_chain():
    """'aa' on a long run of 'a' starting at an odd address: the guessed restart
    phase is wrong in every segment and never meets the truth, so one repair
    walks the whole haystack."""
    pats = [b"aa"]
    im = ii.Image(pats, 0)
    orc = Oracle(pats, "Standard")
    for lead in (0, 1, 3):
        hay = b"b" * lead + b"a" * 700
        st_ = {}
        assert ii.find_staged(im, hay, segment_bytes=128, stats=st_) == orc.find(hay)
    hays = [b"a" * 301, b"", b"a" * 299, b"ba" * 200]
    data, offs = batch(hays)
    assert ii.emulate_scan(im, data, offs, segment_bytes=128, base_addr=1) == oracle_batch(orc, hays)


def test_names_automaton_shape_and_parity():
    pats = [l.strip().encode() for l in open(os.path.join(os.path.dirname(HERE), "ahocorasick_rs_b200", "data", "patterns_long.txt"))]
    im = ii.Image(pats, 0, 2)
    assert im.n_states == 11163 + 1          # SURVEY.md section 6: 11 163 trie states (+ the dead state)
    assert im.col_mode == 0 and im.n_cols == 27 and im.col_lo == ord("a")
    line = ("no one who had ever seen charlotte in her infancy would have supposed her born to be an heroine. "
            "her name was whatevs—and isabella had never been handsome 12345. " * 6).encode()
    orc = Oracle(pats, "Standard")
    exp = orc.find_str(line.decode())
    assert len(exp) >= 12 and ii.find(im, line, cp=True) == exp
    for H in (100, 1200):
        assert ii.find_staged(im, line, cp=True, H=H, base_addr=7, segment_bytes=256) == exp
    for kind in ("LeftmostFirst", "LeftmostLongest"):
        im2 = ii.Image(pats, KID[kind])
        assert ii.find_staged(im2, line, H=1200, segment_bytes=256) == Oracle(pats, kind).find(line)


def test_profiled_hot_set_keeps_results_and_cuts_traps():
    from ahocorasick_rs_b200 import workloads as W
    pats, data, offs = W.config2(3)
    bp = [p.encode() for p in pats]
    im = ii.Image(bp, 0, 2)
    # visit counts as acb_profile would produce them from haystack 0
    visits = np.zeros(im.n_states, dtype=np.uint32)
    s = 1
    for b in bytes(data[offs[0]:offs[1]]):
        e = int(im.trans[s, im.col(b)])
        s = e & ii.MASK
        if e & ii.FLAG:
            s = 1
        visits[s] += 1
    sub, so = data[offs[1]:offs[2]], np.array([0, offs[2] - offs[1]])
    exp = [(0, p, s, e) for (p, s, e) in Oracle(bp, "Standard").find_str(bytes(sub).decode())]
    st_bfs, st_prof = {}, {}
    assert ii.emulate_scan(im, sub, so, cp=True, H=256, stats=st_bfs) == exp
    assert ii.emulate_scan(im, sub, so, cp=True, H=256, stats=st_prof, visits=visits) == exp
    assert st_prof.get("traps", 0) * 20 < st_bfs["traps"]      # 256 profiled rows beat 256 shallowest rows by far
    table, h2f, f2h, rows = im.hot_image(visits, 300)
    assert rows == 300 and h2f[0] == 1 and f2h[1] == 0 and f2h[0] == 0xFFFF
    assert len(set(h2f[:rows].tolist())) == rows and all(f2h[h2f[i]] == i for i in range(rows))


def test_byte_indexed_table_agrees_with_compact_table():
    """For every pattern set with a byte-indexed table -- class columns, range columns ending at 0x7e, range columns
    from 0x00 -- its rows equal the compact table's, byte by byte, and column 127 (where the scan folds every byte
    >= 0x80) equals the compact table's column of each such byte."""
    import struct
    from ahocorasick_rs_b200 import _capi
    from tests.table_shapes import BYTE_TABLE
    sets = [[b"hello", b"help", b"world", b"wor", b"~x"]] + [c.pats for c in BYTE_TABLE]
    seen = set()
    for pats in sets:
        for kind in range(3):
            im = ii.Image(pats, kind)
            seen.add((im.col_mode, max(b for p in pats for b in p) == 0x7E, im.col_lo == 0))
            L = im._L
            n = L.acb_hot_bytes(im._h, 40)
            buf = np.zeros(n, dtype=np.uint8)
            assert L.acb_hot_build(im._h, None, 40, buf.ctypes.data, n) == 0
            desc = _capi.HotDesc()
            assert L.acb_hot_describe(buf.ctypes.data, __import__("ctypes").byref(desc)) == 0
            assert desc.rows == min(40, im.n_states - 1) and desc.rows128 == desc.rows and desc.visited == 1
            magic, rows, n_cols, n_states, o_t, o_h2f, o_f2h, total, rows128, visited, o_t128 = struct.unpack_from("<4I4Q2IQ", buf.tobytes()[:64])
            t = buf[o_t:o_t + 2 * (rows + 1) * n_cols].view(np.uint16).reshape(rows + 1, n_cols) // (2 * n_cols)
            t128 = buf[o_t128:o_t128 + 2 * (rows128 + 1) * 128].view(np.uint16).reshape(rows128 + 1, 128) // 256
            for h in range(rows128 + 1):
                for b in range(128):
                    assert t128[h, b] == t[h, im.col(b)]
                for b in range(128, 256):
                    assert t128[h, 127] == t[h, im.col(b)]
    assert {(1, True, False), (0, True, False), (0, False, True)} <= seen
    # a pattern byte >= 0x7f rules the byte-indexed table out
    im = ii.Image([b"caf\xc3\xa9"], 0)
    n = im._L.acb_hot_bytes(im._h, 40)
    buf = np.zeros(n, dtype=np.uint8)
    assert im._L.acb_hot_build(im._h, None, 40, buf.ctypes.data, n) == 0
    desc = _capi.HotDesc()
    im._L.acb_hot_describe(buf.ctypes.data, __import__("ctypes").byref(desc))
    assert desc.rows128 == 0


def test_builder_errors():
    with pytest.raises(ValueError):
        ii.Image([b"a", b""])
    im = ii.Image([b"ab", b"ab", b"b"], 0)
    assert ii.find(im, b"xab") == [(0, 1, 3)]
    assert ii.find(im, b"xab", overlapping=True) == [(0, 1, 3), (1, 1, 3), (2, 2, 3)]
