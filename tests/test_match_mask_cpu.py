"""Match masks without a GPU: a Python model of the sieve's cover mode (scan_sieve.cuh, kSieveCover) over the chains of
the sieve-image interpreter, checked against the union of the brute-force statement's spans; the C ABI's argument
checks and exports; the Python argument errors; and the host decoding of spans from packed words."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi
from ahocorasick_rs_b200.matcher import spans_from_words

from .sieve_interp import SieveImage
from .spec_bruteforce import spec_find


# ---- the cover rule: at each end position, the deepest (admitted) terminal node's span covers every match ending there
def model_cover(img, text, hs, he, S=None):
    """The bytes [hs, he) the cover mode sets: for every end e, [e - depth, e) of the first admitted entry of the chain
    (longest first), as stage 2 takes best_d."""
    cov = np.zeros(len(text), dtype=bool)
    for e in range(hs + 1, he + 1):
        for pid, start in img.matches_ending_at(text, e, hs):
            if S is None or pid in S:
                cov[start:e] = True
                break
    return cov


def spec_cover(patterns, text, hs, he, kind="Standard", overlapping=True, S=None):
    """The union of [start, end) over the records of the brute-force statement, as a byte mask of text."""
    cov = np.zeros(len(text), dtype=bool)
    for _, a, e in spec_find(patterns, text[hs:he], kind, overlapping, admitted=S):
        cov[hs + a:hs + e] = True
    return cov


@pytest.mark.parametrize("seed", range(8))
def test_cover_model_equals_union_of_spans(seed):
    rng = random.Random(seed)
    alpha = b"ab" if seed % 2 else b"abc"
    pats = [bytes(rng.choice(alpha) for _ in range(rng.randint(1, 6))) for _ in range(rng.randint(2, 12))]
    pats += [pats[0], b"abcab", b"bcab", b"cab", b"ab"]   # a duplicate and a nested family
    img = SieveImage(pats, 0)
    for _ in range(5):
        hays = [bytes(rng.choice(alpha) for _ in range(rng.randint(0, 50))) for _ in range(4)]
        text = b"".join(hays)
        offs = np.concatenate([[0], np.cumsum([len(h) for h in hays])])
        for S in (None, {p for p in range(len(pats)) if rng.random() < 0.4}, set()):
            for h in range(len(hays)):
                hs, he = int(offs[h]), int(offs[h + 1])
                assert np.array_equal(model_cover(img, text, hs, he, S), spec_cover(pats, text, hs, he, S=S)), (h, S)


def test_cover_unadmitted_long_pattern_over_admitted_short_one():
    pats = [b"abcd", b"cd", b"bcd"]
    img = SieveImage(pats, 0)
    text = b"xabcdx"
    for S, want in (({1}, [3, 5]), ({0}, [1, 5]), ({1, 2}, [2, 5]), (set(), None)):
        cov = model_cover(img, text, 0, len(text), S)
        assert np.array_equal(cov, spec_cover(pats, text, 0, len(text), S=S))
        assert (np.flatnonzero(cov).tolist() == list(range(*want))) if want else not cov.any()


@pytest.mark.parametrize("kind", ["Standard", "LeftmostFirst", "LeftmostLongest"])
def test_non_overlapping_cover_is_a_subset_of_the_overlapping_one(kind):
    """The epilogue ORs the selection's spans: a subset of the overlapping cover, and equal to it where matches do not
    overlap.  (The statement's union is what the GPU tests compare against.)"""
    rng = random.Random(len(kind))
    pats = [b"ab", b"abab", b"ba", b"b"]
    for _ in range(20):
        text = bytes(rng.choice(b"ab") for _ in range(rng.randint(0, 40)))
        sel = spec_cover(pats, text, 0, len(text), kind, overlapping=False)
        over = spec_cover(pats, text, 0, len(text), "Standard", overlapping=True)
        assert not (sel & ~over).any()


# ---- the C ABI -------------------------------------------------------------------------------------------------------
MASK_CALLS = ["acb_match_mask_overlapping", "acb_match_mask_overlapping_filtered", "acb_match_mask_non_overlapping",
              "acb_match_mask_non_overlapping_filtered", "acb_mask_rows", "acb_mask_unpack"]


def test_exports():
    L = _capi.lib()
    for name in MASK_CALLS:
        assert name in _capi.EXPORTS
        assert hasattr(L, name)


def _automaton(kind=0, patterns=(b"ab", b"b")):
    L = _capi.lib()
    pats = list(patterns)
    offs = np.zeros(len(pats) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in pats], out=offs[1:])
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, len(pats), kind, -1, C.byref(h)) == 0
    return L, h


def _workspace(null=None):
    ws = _capi.Workspace()
    for name, t in ws._fields_:
        setattr(ws, name, 0x4000 if t is C.c_void_p else 1024)
    if null:
        setattr(ws, null, None)
    return ws


P = 0x3000   # never dereferenced: every refusal below happens before any device work


@pytest.mark.parametrize("bad", ["a", "sieve", "offsets", "mask", "scratch", "bytes", "n_low", "n_high", "total"])
def test_overlapping_einval(bad):
    L, h = _automaton()
    try:
        args = dict(a=h, sieve=P, bytes=P, offsets=P, n=1, total=16, mask=P, scratch=P)
        if bad in ("a", "sieve", "offsets", "mask", "scratch", "bytes"):
            args[bad] = None
        elif bad == "n_low":
            args["n"] = -1
        elif bad == "n_high":
            args["n"] = 0xFFFFFFFF
        else:
            args["total"] = 1 << 31
        for fn, extra in ((L.acb_match_mask_overlapping, ()), (L.acb_match_mask_overlapping_filtered, (None,))):
            rc = fn(args["a"], args["sieve"], args["bytes"], args["offsets"], args["n"], args["total"], args["mask"], 7, args["scratch"],
                    *extra, None)
            assert rc == _capi.ACB_EINVAL, (bad, _capi.last_error())
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("bad", ["a", "sieve", "offsets", "mask", "plan", "bytes", "ws", "ws_raw", "ws_out", "n_high", "total", "plan_shape"])
def test_non_overlapping_einval(bad):
    L, h = _automaton()
    try:
        plan = _capi.Plan()
        assert L.acb_plan_scan(h, P, 16, 1, C.byref(plan)) == 0
        if bad == "plan_shape":
            plan.n_units += 1
        ws = _workspace({"ws_raw": "dev_raw", "ws_out": "dev_out"}.get(bad))
        args = dict(a=h, sieve=P, bytes=P, offsets=P, n=1, total=16, mask=P, plan=C.byref(plan), ws=C.byref(ws))
        if bad in ("a", "sieve", "offsets", "mask", "plan", "bytes", "ws"):
            args[bad] = None
        elif bad == "n_high":
            args["n"] = 0xFFFFFFFF
        elif bad == "total":
            args["total"] = 1 << 31
        for fn, extra in ((L.acb_match_mask_non_overlapping, ()), (L.acb_match_mask_non_overlapping_filtered, (None,))):
            rc = fn(args["a"], args["sieve"], args["bytes"], args["offsets"], args["n"], args["total"], args["plan"], args["ws"],
                    args["mask"], 7, *extra, None)
            assert rc == _capi.ACB_EINVAL, (bad, _capi.last_error())
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("bad", ["no_sets", "null_bits", "index_bytes", "null_index"])
def test_filter_einval(bad):
    L, h = _automaton()
    try:
        f = _capi.PatternFilter()
        f.dev_set_bits, f.n_sets, f.dev_set_index, f.index_bytes = 0x1000, 1, 0x2000, 4
        if bad == "no_sets":
            f.n_sets = 0
        elif bad == "null_bits":
            f.dev_set_bits = None
        elif bad == "index_bytes":
            f.index_bytes = 8 + 1
        else:
            f.dev_set_index = None
        plan = _capi.Plan()
        assert L.acb_plan_scan(h, P, 16, 1, C.byref(plan)) == 0
        ws = _workspace()
        assert L.acb_match_mask_overlapping_filtered(h, P, P, P, 1, 16, P, 0, P, C.byref(f), None) == _capi.ACB_EINVAL
        assert L.acb_match_mask_non_overlapping_filtered(h, P, P, P, 1, 16, C.byref(plan), C.byref(ws), P, 0, C.byref(f), None) == _capi.ACB_EINVAL
        assert "pattern filter" in _capi.last_error()
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [1, 2])
def test_overlapping_on_leftmost_is_unsupported(kind):
    """Refused before any byte is read: the sieve image need not even exist."""
    L, h = _automaton(kind)
    try:
        assert L.acb_match_mask_overlapping(h, P, P, P, 1, 16, P, 0, P, None) == _capi.ACB_EUNSUPPORTED
        assert L.acb_match_mask_overlapping_filtered(h, P, P, P, 1, 16, P, 0, P, None, None) == _capi.ACB_EUNSUPPORTED
        assert "does not support overlapping" in _capi.last_error()
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("bad", ["rows", "offsets", "mask", "row_bytes", "n_low", "n_high"])
def test_mask_rows_einval(bad):
    L = _capi.lib()
    args = dict(rows=P, row_bytes=8, n_rows=3, offsets=P, n=1, mask=P)
    if bad in ("rows", "offsets", "mask"):
        args[bad] = None
    elif bad == "row_bytes":
        args["row_bytes"] = 16
    elif bad == "n_low":
        args["n"] = -1
    else:
        args["n"] = 0xFFFFFFFF
    rc = L.acb_mask_rows(args["rows"], args["row_bytes"], args["n_rows"], args["offsets"], args["n"], args["mask"], 0, None)
    assert rc == _capi.ACB_EINVAL


@pytest.mark.parametrize("bad", ["mask", "out", "stride"])
def test_mask_unpack_einval(bad):
    L = _capi.lib()
    args = dict(mask=P, stride=1, out=P)
    args[bad] = 0 if bad == "stride" else None
    assert L.acb_mask_unpack(args["mask"], 0, args["stride"], 10, args["out"], None) == _capi.ACB_EINVAL


# ---- Python argument errors --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [MatchKind.LeftmostFirst, MatchKind.LeftmostLongest])
def test_overlapping_on_leftmost_raises(kind):
    data, offs = torch.zeros(4, dtype=torch.uint8), torch.tensor([0, 4])
    for ac, hay in ((BytesAhoCorasick([b"ab"], matchkind=kind), b"ab"), (AhoCorasick(["ab"], matchkind=kind), "ab"),
                    (TokenAhoCorasick([[1, 2]], matchkind=kind), [1, 2])):
        with pytest.raises(ValueError, match="does not support overlapping"):
            ac.match_mask_device(data, offs, True)
        with pytest.raises(ValueError, match="does not support overlapping"):
            ac.match_spans(hay, overlapping=True)
        with pytest.raises(ValueError, match="does not support overlapping"):
            ac.match_spans_batch([hay], overlapping=True)


def test_argument_errors():
    ac = BytesAhoCorasick([b"ab"])
    data, offs = torch.zeros(4, dtype=torch.uint8), torch.tensor([0, 4])
    ps = ac.pattern_sets([[0]], device="cpu")
    with pytest.raises(ValueError, match="together"):
        ac.match_mask_device(data, offs, pattern_sets=ps)
    with pytest.raises(ValueError, match="shape"):
        ac.match_mask_device(data, offs, pattern_sets=ps, set_index=torch.zeros(2, dtype=torch.int32))
    with pytest.raises(TypeError):
        ac.match_spans("ab")
    with pytest.raises(TypeError):
        AhoCorasick(["ab"]).match_spans(b"ab")
    with pytest.raises(TypeError):
        AhoCorasick(["ab"]).match_spans_batch(["ab", b"ab"])
    for a, hays in ((ac, [b"x", b"y"]), (AhoCorasick(["ab"]), ["x", "y"]), (TokenAhoCorasick([[1, 2]]), [[1], [2]])):
        with pytest.raises(ValueError, match="one set of pattern ids per haystack"):
            a.match_spans_batch(hays, patterns=[[0]])
    tac = TokenAhoCorasick([[1, 2]])
    with pytest.raises(TypeError, match="int64 tensor of token offsets"):
        tac.match_mask_device(torch.zeros(4, dtype=torch.int64), [0, 4])
    with pytest.raises(ValueError, match="outside"):
        tac.match_spans([1, 1 << 21])


# ---- host decoding of spans from packed words ----------------------------------------------------------------------
def _spans_of(bits, offs, text=None, unit=1):
    """The straightforward decoding: per haystack, runs of covered positions, mapped to code points by counting lead
    bytes, or divided by unit."""
    out = []
    for h in range(len(offs) - 1):
        hs, he = offs[h], offs[h + 1]
        pos = (lambda b: sum(1 for c in text[hs:b] if c & 0xC0 != 0x80)) if text is not None else (lambda b: (b - hs) // unit)
        runs, p = [], hs
        while p < he:
            if bits[p]:
                q = p
                while q < he and bits[q]:
                    q += 1
                runs.append((pos(p), pos(q)))
                p = q
            else:
                p += 1
        out.append(runs)
    return out


def _pack(bits):
    words = np.zeros((len(bits) + 31) // 32 + 1, dtype=np.uint32)
    for p in np.flatnonzero(bits):
        words[p // 32] |= np.uint32(1 << (p % 32))
    return words.view(np.int32)


@pytest.mark.parametrize("cut", range(33))
def test_boundaries_at_every_bit_of_a_word(cut):
    """Two haystacks meeting at bit `cut` of word 1, with a run across the boundary: the run is cut there."""
    total = 96
    offs = np.array([0, 32 + cut, total], dtype=np.int64)
    bits = np.zeros(total, dtype=bool)
    bits[20:80] = True
    bits[90:96] = True
    got = spans_from_words(_pack(bits), offs)
    assert got == _spans_of(bits, offs)
    assert got[0][-1] == (20, 32 + cut) and got[1][0] == (0, 80 - 32 - cut)


@pytest.mark.parametrize("seed", range(10))
def test_random_layouts(seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 70, size=rng.integers(1, 30))
    offs = np.concatenate([[int(rng.integers(0, 40))], lens]).cumsum()
    total = int(offs[-1])
    bits = rng.random(total) < rng.choice([0.1, 0.5, 0.9])
    got = spans_from_words(_pack(bits), offs)
    bits[:offs[0]] = False
    assert got == _spans_of(bits, offs)
    assert got == spans_from_words(_pack(bits), offs)   # bytes before offs[0] never count


@pytest.mark.parametrize("seed", range(6))
def test_code_points(seed):
    """2-4-byte code points: a covered code point has every byte covered, and positions count lead bytes."""
    rng = random.Random(seed)
    alpha = ["a", "é", "€", "😀", "b"]
    hays = ["".join(rng.choice(alpha) for _ in range(rng.randint(0, 25))) for _ in range(12)]
    enc = [h.encode() for h in hays]
    text = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)[:sum(len(e) for e in enc)]
    offs = np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.int64)
    bits = np.zeros(len(text), dtype=bool)
    want = []
    for h, s in enumerate(hays):
        cov = [rng.random() < 0.5 for _ in s]
        pos = int(offs[h])
        for c, on in zip(s, cov):
            n = len(c.encode())
            bits[pos:pos + n] = on
            pos += n
        runs, i = [], 0
        while i < len(s):
            if cov[i]:
                j = i
                while j < len(s) and cov[j]:
                    j += 1
                runs.append((i, j))
                i = j
            else:
                i += 1
        want.append(runs)
    assert spans_from_words(_pack(bits), offs, text) == want


def test_token_unit():
    offs = np.array([0, 9, 18], dtype=np.int64)
    bits = np.zeros(18, dtype=bool)
    bits[3:9] = True    # tokens 1-2 of haystack 0
    bits[9:12] = True   # token 0 of haystack 1
    assert spans_from_words(_pack(bits), offs, unit=3) == [[(1, 3)], [(0, 1)]]
