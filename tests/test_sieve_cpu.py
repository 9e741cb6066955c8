"""CPU checks of the sieve image (csrc/sieve.cpp) and of the sieve scan's logic
(tests/sieve_interp.py follows scan_sieve.cuh and the epilogue's selection)
against the oracle: every match kind, overlapping, duplicates, tiny alphabets
(dense suffix sharing), short patterns (W < 4), long patterns (W > 4), a
filter that is far too small (everything falls through to the exact check)."""
import numpy as np
import pytest

from oracle import Oracle
from tests.sieve_inputs import FANOUTS, TWO_LEVEL, fanout_case
from tests.sieve_interp import SieveImage, scan
from ahocorasick_rs_b200 import workloads as W

KINDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def oracle_rows(pats, kind, data, offs, overlapping):
    total, counts, rec = Oracle(pats, kind).scan_batch(np.asarray(data, dtype=np.uint8), np.asarray(offs, dtype=np.int64),
                                                       overlapping=overlapping)
    return [tuple(int(x) for x in r) for r in rec]


def random_case(rng, alphabet, n_pat, lo, hi, n_hay, max_hay):
    al = np.frombuffer(alphabet, dtype=np.uint8)
    pats = [bytes(al[rng.integers(0, len(al), size=int(rng.integers(lo, hi + 1)))]) for _ in range(n_pat)]
    lens = rng.integers(0, max_hay + 1, size=n_hay)
    data = al[rng.integers(0, len(al), size=int(lens.sum()))].astype(np.uint8)
    offs = np.zeros(n_hay + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    return pats, data, offs


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("shape", [(b"ab", 12, 1, 4), (b"abc", 40, 1, 9), (b"abcd", 60, 4, 7), (b"ab", 30, 5, 12),
                                   (b"abcdefgh", 200, 5, 8), (b"xy", 25, 8, 20)])
def test_interpreter_matches_oracle(kind, shape):
    alphabet, n_pat, lo, hi = shape
    rng = np.random.default_rng(1000 * kind + n_pat)
    for rep in range(3):
        pats, data, offs = random_case(rng, alphabet, n_pat, lo, hi, n_hay=12, max_hay=120)
        img = SieveImage(pats, kind)
        assert img.W == min(min(len(p) for p in pats), img.W) and img.W <= 8
        for overlapping in ([False, True] if kind == 0 else [False]):
            assert scan(img, data, offs, overlapping) == oracle_rows(pats, KINDS[kind], data, offs, overlapping)


@pytest.mark.parametrize("w_max", [1, 2, 3, 4, 5, 6, 7, 8])
def test_forced_window_sizes(w_max):
    rng = np.random.default_rng(77 + w_max)
    pats, data, offs = random_case(rng, b"abc", 80, 8, 14, n_hay=6, max_hay=300)
    img = SieveImage(pats, 0, w_max=w_max)
    assert img.W == w_max
    assert scan(img, data, offs, True) == oracle_rows(pats, "Standard", data, offs, True)
    assert scan(img, data, offs, False) == oracle_rows(pats, "Standard", data, offs, False)


def test_tiny_filter_still_exact():
    """1 KiB of filter for 3 000 patterns: nearly every position passes it; the exact check decides."""
    rng = np.random.default_rng(5)
    pats, data, offs = random_case(rng, b"abcdef", 3000, 4, 9, n_hay=4, max_hay=400)
    img = SieveImage(pats, 2, bloom_bytes_max=1024)
    assert img.last_level == img.W
    assert scan(img, data, offs, False) == oracle_rows(pats, "LeftmostLongest", data, offs, False)


@pytest.mark.parametrize("w_max", [1, 5, 8])
@pytest.mark.parametrize("fanout", list(FANOUTS) + [TWO_LEVEL])
def test_trie_fanout(fanout, w_max):
    """A trie node with 1, 8, 9, 255 or 256 children (and two levels of many), every byte value before it in the text:
    the builder's child lists (sorted, 9-bit counts) give the oracle's matches for every kind."""
    pats, data, offs = fanout_case(fanout)
    for kind in range(3):
        img = SieveImage(pats, kind, w_max=w_max)
        assert img.W == w_max
        for overlapping in ([False, True] if kind == 0 else [False]):
            assert scan(img, data, offs, overlapping) == oracle_rows(pats, KINDS[kind], data, offs, overlapping)


def test_fanout_inputs_reach_their_child_counts():
    """The node of the core has exactly the children asked for (the count of 256 needs the 9th bit of the field)."""
    for fanout in list(FANOUTS) + [TWO_LEVEL]:
        pats, _, _ = fanout_case(fanout)
        img = SieveImage(pats, 0, w_max=8)
        counts = (img.na[: img.n_nodes, 1] >> 8) & 0x1FF
        assert counts.max() == (12 if fanout == TWO_LEVEL else fanout), fanout
        if fanout == TWO_LEVEL:
            assert (counts == 10).sum() == 12


def test_duplicates_nested_and_self_overlapping():
    pats = [b"a", b"aa", b"aaa", b"a", b"aa", b"ba", b"ab", b"aab", b"b"]
    data = np.frombuffer(b"aaaabaaabbbaabaaaa", dtype=np.uint8)
    offs = np.array([0, 7, 7, 12, len(data)], dtype=np.int64)
    for kind in range(3):
        img = SieveImage(pats, kind)
        for overlapping in ([False, True] if kind == 0 else [False]):
            assert scan(img, data, offs, overlapping) == oracle_rows(pats, KINDS[kind], data, offs, overlapping)


def test_reference_shapes_filter_quality():
    """On the config-2 shape the on-chip levels should leave almost nothing but true matches for the exact check."""
    pats, data, offs = W.config2(6)
    pb = [p.encode() for p in pats]
    img = SieveImage(pb, 0)
    rows = scan(img, data, offs, False)
    assert rows == oracle_rows(pb, "Standard", data, offs, False)
    st = img.stats
    assert st["stage2"] * 100 <= st["pos"], st   # under 1 % of the positions leave the SM
    assert img.last_level > img.W


def test_high_bytes_and_binary_patterns():
    rng = np.random.default_rng(9)
    pats = [bytes(rng.integers(0, 256, size=int(rng.integers(1, 7)), dtype=np.uint8)) for _ in range(50)]
    data = rng.integers(0, 256, size=3000, dtype=np.uint8)
    for p in pats[:20]:
        at = int(rng.integers(0, len(data) - len(p)))
        data[at:at + len(p)] = np.frombuffer(p, dtype=np.uint8)
    offs = np.array([0, 1000, 3000], dtype=np.int64)
    img = SieveImage(pats, 0)
    assert scan(img, data, offs, True) == oracle_rows(pats, "Standard", data, offs, True)


def test_filters_leave_room_for_a_deeper_ring_on_sparse_sets():
    """csrc/sieve.cpp: the builder gives up filter bytes for a deeper ring of text per warp (24 warps x 576 B per extra
    window) while that cuts the estimated stage-1 rounds per window by a quarter or more; dense sets keep every byte."""
    budget = 232448 - 46 * 1024
    slot = 24 * 576
    rng = np.random.default_rng(7)
    al = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)

    def pats(n, lo, hi):
        return [bytes(al[rng.integers(0, 26, size=int(rng.integers(lo, hi + 1)))]) for _ in range(n)]

    dense = SieveImage(pats(50_000, 5, 12), 0, budget)          # ~50 k keys: chance survivors fill a round per window
    assert budget - slot < dense.bloom_words * 4 <= budget
    mid = SieveImage(pats(10_000, 5, 12), 0, budget)            # ~10 k keys: a ring of four windows
    assert budget - 4 * slot < mid.bloom_words * 4 <= budget - 3 * slot
    few = SieveImage(pats(2_000, 5, 12), 0, budget)             # a ring of eight
    assert few.bloom_words * 4 <= budget - 7 * slot
    # the primary bitmap stays the sparse part: at most one bit in 64 set by chance on the sparse sets
    assert few.n_keys * 64 <= few.prim_words * 32 and mid.n_keys * 64 <= mid.prim_words * 32
