"""Pattern sets without a GPU: the bitset packing, every argument error, the C ABI's filter checks and exports, and a
Python model of the sieve's admitted-pid rules (scan_sieve.cuh, SieveFilter) over the chains of the sieve-image
interpreter, checked against automata built from each subset."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi
from ahocorasick_rs_b200.matcher import PatternSets, _filter_args

from .sieve_geometry_helpers import subset_scan_batch
from .sieve_interp import SieveImage
from .spec_bruteforce import spec_find

KINDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def _np_pack(mask):
    G, P = mask.shape
    words = max((P + 31) // 32, 1)
    out = np.zeros((G, words), dtype=np.uint32)
    for g in range(G):
        for p in range(P):
            if mask[g, p]:
                out[g, p // 32] |= np.uint32(1 << (p % 32))
    return out


@pytest.mark.parametrize("P", [1, 31, 32, 33, 70])
def test_pack_from_tensor_matches_numpy(P):
    rng = np.random.default_rng(P)
    mask = rng.random((5, P)) < 0.4
    mask[0] = True
    mask[1] = False
    ac = BytesAhoCorasick([bytes([65 + i % 26]) * (1 + i // 26) for i in range(P)])
    ps = ac.pattern_sets(torch.from_numpy(mask), device="cpu")
    assert ps.n_sets == 5 and ps.words == (P + 31) // 32
    assert np.array_equal(ps.bits.numpy().view(np.uint32), _np_pack(mask))


def test_pack_from_lists_matches_numpy():
    P = 40
    ac = BytesAhoCorasick([b"p%02d" % i for i in range(P)])
    sets = [[0, 31, 32, 39], [], range(P), (5, 5, 7)]
    mask = np.zeros((len(sets), P), dtype=bool)
    for g, s in enumerate(sets):
        mask[g, list(s)] = True
    ps = ac.pattern_sets(sets, device="cpu")
    assert np.array_equal(ps.bits.numpy().view(np.uint32), _np_pack(mask))


@pytest.mark.parametrize("sets", [[[3]], [[-1]], [[0, 1, 2, 3]], [], [["a"]]])
def test_bad_sets_raise(sets):
    ac = BytesAhoCorasick([b"a", b"b", b"c"])
    with pytest.raises(ValueError):
        ac.pattern_sets(sets, device="cpu")


def test_bad_tensor_shapes_raise():
    ac = BytesAhoCorasick([b"a", b"b", b"c"])
    for t in (torch.zeros((2, 4), dtype=torch.bool), torch.zeros(3, dtype=torch.bool), torch.zeros((2, 3), dtype=torch.int32),
              torch.zeros((0, 3), dtype=torch.bool)):
        with pytest.raises(ValueError):
            ac.pattern_sets(t, device="cpu")


def test_filter_argument_checks():
    ac = BytesAhoCorasick([b"a", b"b", b"c"])
    other = BytesAhoCorasick([b"a", b"b", b"c"])
    ps = ac.pattern_sets([[0], [1, 2]], device="cpu")
    dev = torch.device("cpu")
    idx = torch.tensor([0, 1, 1], dtype=torch.int32)
    assert _filter_args(ac._ac, None, None, 3, dev) is None
    got = _filter_args(ac._ac, ps, idx, 3, dev)
    assert got[0] is ps and got[1].dtype == torch.int32
    with pytest.raises(ValueError, match="together"):
        _filter_args(ac._ac, ps, None, 3, dev)
    with pytest.raises(ValueError, match="together"):
        _filter_args(ac._ac, None, idx, 3, dev)
    with pytest.raises(ValueError, match="this automaton"):
        _filter_args(ac._ac, other.pattern_sets([[0]], device="cpu"), idx, 3, dev)
    with pytest.raises(ValueError, match="shape"):
        _filter_args(ac._ac, ps, idx[:2], 3, dev)
    with pytest.raises(ValueError, match="shape"):
        _filter_args(ac._ac, ps, idx.to(torch.int16), 3, dev)
    with pytest.raises(ValueError, match=r"\[0, 2\)"):
        _filter_args(ac._ac, ps, torch.tensor([0, 2, 1]), 3, dev)
    with pytest.raises(ValueError, match=r"\[0, 2\)"):
        _filter_args(ac._ac, ps, torch.tensor([0, -1, 1]), 3, dev)
    with pytest.raises(ValueError, match="live on"):
        _filter_args(ac._ac, ps, idx, 3, torch.device("meta"))


def test_host_batch_length_mismatch_raises():
    for ac, hays in ((BytesAhoCorasick([b"ab"]), [b"x", b"y"]), (AhoCorasick(["ab"]), ["x", "y"]),
                     (TokenAhoCorasick([[1, 2]]), [[1], [2]])):
        for call in (ac.is_match_batch, ac.find_first_batch, ac.count_matches_batch, ac.find_matches_as_indexes_batch):
            with pytest.raises(ValueError, match="one set of pattern ids per haystack"):
                call(hays, patterns=[[0]])


@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_overlapping_on_leftmost_refused_first(kind):
    ac = BytesAhoCorasick([b"ab"], matchkind=kind)
    ps = ac.pattern_sets([[0]], device="cpu")
    data, offs, idx = torch.zeros(4, dtype=torch.uint8), torch.tensor([0, 4]), torch.zeros(1, dtype=torch.int32)
    for call in (ac.scan_device, ac.count_matches_device):
        with pytest.raises(ValueError, match="does not support overlapping"):
            call(data, offs, True, pattern_sets=ps, set_index=idx)
    with pytest.raises(ValueError, match="does not support overlapping"):
        ac.find_matches_as_indexes(b"ab", overlapping=True, patterns=[0])
    with pytest.raises(ValueError, match="does not support overlapping"):
        ac.count_matches(b"ab", overlapping=True, patterns=[0])


def test_exports():
    new = ["acb_scan_batch_filtered", "acb_any_match_filtered", "acb_find_first_filtered", "acb_first_rows_filtered",
           "acb_count_overlapping_filtered", "acb_count_non_overlapping_filtered", "acb_stream_first_resolve_filtered"]
    L = _capi.lib()
    for name in new:
        assert name in _capi.EXPORTS
        assert hasattr(L, name)


def _automaton(patterns=(b"ab", b"b")):
    L = _capi.lib()
    pats = list(patterns)
    offs = np.zeros(len(pats) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pats], out=offs[1:])
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pats), 0, -1, C.byref(h)) == 0
    return L, h


@pytest.mark.parametrize("bad", ["no_sets", "null_bits", "index_bytes", "null_index"])
def test_capi_filter_einval(bad):
    """Malformed descriptors are refused before any device work (the pointers are never dereferenced)."""
    L, h = _automaton()
    try:
        f = _capi.PatternFilter()
        f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = 0x1000, 1, 0x2000, 4
        if bad == "no_sets":
            f.n_sets = 0
        elif bad == "null_bits":
            f.dev_set_bits = None
        elif bad == "index_bytes":
            f.index_bytes = 2
        else:
            f.dev_set_index = None
        fp = C.byref(f)
        p = 0x3000
        assert L.acb_any_match_filtered(h, p, p, p, 1, 16, p, p, fp, None) == _capi.ACB_EINVAL
        assert L.acb_find_first_filtered(h, p, p, p, 1, 16, p, p, fp, None) == _capi.ACB_EINVAL
        assert L.acb_count_overlapping_filtered(h, p, p, p, 1, 16, p, p, fp, None) == _capi.ACB_EINVAL
        assert L.acb_first_rows_filtered(h, p, p, p, 1, p, p, fp, None) == _capi.ACB_EINVAL
        assert "pattern filter" in _capi.last_error()
    finally:
        L.acb_free(h)


# ---- the admitted-pid rules (scan_sieve.cuh stage 2 with a filter), over the interpreter's chains -------------------
def _chain_rows(img, data, hs, he):
    """[(end, [(pid, start), ...] longest first)] for every position of one haystack (haystack-relative)."""
    out = []
    for e in range(hs + 1, he + 1):
        ch = img.matches_ending_at(data, e, hs)
        if ch:
            out.append((e - hs, [(p, s - hs) for p, s in ch]))
    return out


def model_list(chains, S):
    return [(p, s, e) for e, ch in chains for p, s in ch if p in S]


def model_any(chains, S):
    return any(p in S for _, ch in chains for p, _ in ch)


def model_first(chains, S, kind):
    best = None
    for e, ch in chains:
        adm = [(p, s) for p, s in ch if p in S]
        if not adm:
            continue
        p, s = adm[0]    # deepest node with an admitted pid, its lowest admitted pid
        key = {"Standard": (e, -(e - s)), "LeftmostFirst": (s, p), "LeftmostLongest": (s, -e)}[kind]
        if best is None or key < best[0]:
            best = (key, (p, s, e))
    return None if best is None else best[1]


def model_count(chains, S):
    return sum(1 for _, ch in chains for p, _ in ch if p in S)


def _subset_oracle(patterns, S, hay, kind, overlapping=False):
    ids = [p for p in range(len(patterns)) if p in S]
    return [(ids[p], s, e) for p, s, e in spec_find([patterns[i] for i in ids], hay, kind, overlapping)]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("kind", KINDS)
def test_admitted_pid_model_matches_subset_automaton(seed, kind):
    rng = random.Random(seed * 7 + len(kind))
    alpha = b"abc"
    pats = [bytes(rng.choice(alpha) for _ in range(rng.randint(1, 5))) for _ in range(rng.randint(3, 12))]
    pats += [pats[0], pats[1][:1]]   # duplicates and a nested member
    img = SieveImage(pats, KINDS.index(kind))
    for _ in range(6):
        hay = bytes(rng.choice(alpha) for _ in range(rng.randint(0, 60)))
        S = {p for p in range(len(pats)) if rng.random() < rng.choice([0.0, 0.3, 0.7, 1.0])}
        chains = _chain_rows(img, hay, 0, len(hay))
        over = sorted(model_list(chains, S), key=lambda m: (m[2], m[1], m[0]))
        if kind == "Standard":
            assert over == _subset_oracle(pats, S, hay, kind, True)
            assert model_count(chains, S) == len(over)
        want = _subset_oracle(pats, S, hay, kind)
        assert model_any(chains, S) == bool(want)
        assert model_first(chains, S, kind) == (want[0] if want else None)


def test_model_nested_family_longest_not_allowed():
    pats = [b"abcd", b"bcd", b"cd", b"d"]
    img = SieveImage(pats, 0)
    chains = _chain_rows(img, b"xabcd", 0, 5)
    assert model_first(chains, {1, 3}, "Standard") == (1, 2, 5)
    assert model_first(chains, {3}, "LeftmostLongest") == (3, 4, 5)


def test_model_duplicates_lowest_allowed_id():
    pats = [b"ab", b"ab", b"ab"]
    img = SieveImage(pats, 1)
    chains = _chain_rows(img, b"zab", 0, 3)
    assert model_first(chains, {2, 1}, "LeftmostFirst") == (1, 1, 3)
    assert model_list(chains, {0, 2}) == [(0, 1, 3), (2, 1, 3)]


# ---- subset_scan_batch (the GPU tests' reference) against the brute-force statement --------------------------------
@pytest.mark.parametrize("codepoints", [False, True], ids=["bytes", "str"])
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("search", ["Standard", "LeftmostFirst", "LeftmostLongest", "Overlapping"])
def test_subset_scan_batch_matches_restricted_spec(search, seed, codepoints):
    """subset_scan_batch groups haystacks by set and scans each group with an oracle of that set's patterns; the
    semantics is spec_find on the full list with the occurrences restricted to S (the order is kept, so that is all a
    subset changes).  Duplicates and a nested family; an index outside [0, G) admits nothing."""
    kind, overlapping = ("Standard", True) if search == "Overlapping" else (search, False)
    rng = random.Random(100 * seed + len(search) + codepoints)
    alpha = ["a", "b", "c", "é", "€"] if codepoints else ["a", "b", "c"]
    pats = ["".join(rng.choice(alpha) for _ in range(rng.randint(1, 5))) for _ in range(14)]
    pats += [pats[2], pats[2], "abca", "bca", "ca", "a"]   # duplicates, a nested family
    pb = [p.encode() for p in pats]
    P = len(pats)
    sets = [[], list(range(P)), [P - 3, P - 1], [3, 2, 15]] + [[p for p in range(P) if rng.random() < f] for f in (0.2, 0.6)]
    hays = ["".join(rng.choice(alpha) for _ in range(rng.choice([0, 1, 7, 40, 120]))) for _ in range(30)]
    idx = [rng.randrange(-1, len(sets) + 1) for _ in hays]
    data = np.frombuffer("".join(hays).encode() or b"\0", dtype=np.uint8)[:len("".join(hays).encode())]
    offs = np.zeros(len(hays) + 1, dtype=np.int64)
    np.cumsum([len(h.encode()) for h in hays], out=offs[1:])
    total, counts, rec = subset_scan_batch(pb, kind, data, offs, sets, idx, overlapping, codepoints)
    assert rec.dtype == np.uint32 and rec.shape == (total, 4) and int(counts.sum()) == total
    want_total = 0
    for h, hay in enumerate(hays):
        S = set(sets[idx[h]]) if 0 <= idx[h] < len(sets) else set()
        want = spec_find(pats if codepoints else pb, hay if codepoints else hay.encode(), kind, overlapping, admitted=S)
        got = [tuple(int(x) for x in r[1:]) for r in rec[rec[:, 0] == h]]
        assert got == want, (h, S)
        assert counts[h] == len(want)
        want_total += len(want)
    assert want_total == total and want_total > 0
    assert np.array_equal(rec[:, 0], np.sort(rec[:, 0]))   # haystack order, as Oracle.scan_batch
