"""CPU tests: the C-ABI library loads and exports every symbol include/acb200.h
declares; host-side API behaviour that needs no GPU (construction, argument
and error handling mirrored from the reference's tests)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ahocorasick_rs_b200 import (AhoCorasick, BytesAhoCorasick, Implementation, MatchKind, MATCHKIND_STANDARD,
                                 MATCHKIND_LEFTMOST_FIRST, MATCHKIND_LEFTMOST_LONGEST, _capi)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "acb200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(acb_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 18
    L = _capi.lib()
    for name in declared:
        assert getattr(L, name) is not None, name
    assert declared == set(_capi.EXPORTS)
    assert b"sm_90a" in L.acb_version()


H100_SMEM_OPTIN = 232_448   # opt-in shared memory per block on an H100 (227 KiB)


def sieve_smem(bloom_bytes, ring):
    """scan_sieve.cuh sieve_smem_bytes: the filters, the mbarrier (16 B), then per warp (24) a ring of 576-byte slots
    (16 B of history, a 512-byte window, 48 B of code point counts), a 16-byte pad and two 64-entry queues (4 B, 16 B)."""
    return bloom_bytes + 16 + 24 * (ring * (16 + 512 + 48) + 16 + 64 * 4 + 64 * 16)


def test_sieve_ring_export():
    L = _capi.lib()
    assert "acb_sieve_ring" in _capi.EXPORTS and L.acb_sieve_ring is not None
    assert [f[0] for f in _capi.Tuning._fields_][-1] == "sieve_ring"


@pytest.mark.parametrize("ring,largest", [(8, 90_736), (4, 146_032), (2, 173_680), (1, 187_504)])
def test_sieve_ring_at_its_boundaries(ring, largest):
    """The deepest ring that fits next to the filters, for each of the four depths: at the largest filter that leaves
    room for it, and one byte past it (the next smaller ring, or 0 when not even one window fits)."""
    L = _capi.lib()
    _capi.set_tuning()
    assert sieve_smem(largest, ring) == H100_SMEM_OPTIN
    assert L.acb_sieve_ring(largest, H100_SMEM_OPTIN) == ring
    assert L.acb_sieve_ring(largest + 1, H100_SMEM_OPTIN) == ring // 2
    assert L.acb_sieve_ring(largest - 16, H100_SMEM_OPTIN) == ring
    assert L.acb_sieve_ring(4096, H100_SMEM_OPTIN) == 8
    assert L.acb_sieve_ring(0xFFFF_FFF0, H100_SMEM_OPTIN) == 0


@pytest.mark.parametrize("bloom_bytes,fits", [(4096, 8), (90_736, 8), (90_737, 4), (146_033, 2), (173_681, 1)])
def test_sieve_ring_cap_rounds_down_and_never_raises(bloom_bytes, fits):
    L = _capi.lib()
    try:
        for cap in range(0, 20):
            _capi.set_tuning(5, 0, 512, 0, sieve_ring=cap)
            want = fits if cap == 0 else min(fits, 1 << (cap.bit_length() - 1))
            assert L.acb_sieve_ring(bloom_bytes, H100_SMEM_OPTIN) == want, cap
        _capi.set_tuning(sieve_ring=3)
        assert L.acb_sieve_ring(4096, H100_SMEM_OPTIN) == 2
        _capi.set_tuning(sieve_ring=9)
        assert L.acb_sieve_ring(4096, H100_SMEM_OPTIN) == 8
        _capi.set_tuning(sieve_ring=-1)   # not a cap: as many as fit
        assert L.acb_sieve_ring(bloom_bytes, H100_SMEM_OPTIN) == fits
    finally:
        _capi.set_tuning()
    assert L.acb_sieve_ring(bloom_bytes, H100_SMEM_OPTIN) == fits


def test_build_and_image_roundtrip_without_gpu():
    L = _capi.lib()
    pats = [b"hello", b"world", b"fish"]
    offs = np.array([0, 5, 10, 14], dtype=np.uint64)
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, 3, 0, -1, C.byref(h)) == 0
    assert L.acb_num_patterns(h) == 3 and L.acb_max_pattern_len(h) == 5 and L.acb_min_pattern_len(h) == 4
    assert L.acb_num_states(h) == 2 + 14
    n = L.acb_image_bytes(h)
    buf = np.zeros(n, dtype=np.uint8)
    assert L.acb_image_write(h, buf.ctypes.data, n - 1) == _capi.ACB_ECAPACITY
    assert L.acb_image_write(h, buf.ctypes.data, n) == 0
    L.acb_free(h)
    bad = np.array([0, 5, 5, 14], dtype=np.uint64)  # an empty pattern
    assert L.acb_build(blob.ctypes.data, bad.ctypes.data, 3, 0, -1, C.byref(h)) == _capi.ACB_EBUILD
    assert b"empty pattern" in L.acb_last_error()
    plan = _capi.Plan()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, 3, 0, -1, C.byref(h)) == 0
    assert L.acb_plan_scan(h, 64 + 5, 409_600_000, 100_000, C.byref(plan)) == 0
    assert plan.segment_bytes == 1024 and plan.warm_bytes == 16 and plan.lane_stride == 4
    assert plan.n_segments == (409_600_000 + 5 + 1023) // 1024 and plan.n_units == 2 * plan.n_segments
    assert plan.scratch_words > plan.n_segments
    assert L.acb_plan_scan(h, 0, 1 << 20, 1, C.byref(plan)) == 0 and plan.lane_stride == 1
    L.acb_free(h)


def test_constructor_errors_like_the_reference():
    # reference tests/test_ac.py:75-83, 157-168; tests/test_ac_bytes.py:118-130, 164-172
    with pytest.raises(TypeError):
        AhoCorasick(None)
    with pytest.raises(TypeError):
        AhoCorasick(["x", 12])
    for bad in ([""], ["", "xx"], ["xx", ""]):
        for sp in (True, False):
            with pytest.raises(ValueError) as e:
                AhoCorasick(bad, store_patterns=sp)
            assert "You passed in an empty string as a pattern" in str(e.value)
    with pytest.raises(TypeError):
        BytesAhoCorasick(None)
    with pytest.raises(TypeError):
        BytesAhoCorasick([b"x", 12])
    with pytest.raises(TypeError):
        BytesAhoCorasick([b"x", "y"])
    for bad in ([b""], [b"", b"xx"], [b"xx", b""]):
        with pytest.raises(ValueError) as e:
            BytesAhoCorasick(bad)
        assert "You passed in an empty pattern" in str(e.value)
    with pytest.raises(TypeError):
        BytesAhoCorasick([np.zeros((2, 2), dtype=np.uint8)])  # more than one dimension
    with pytest.raises(TypeError):
        BytesAhoCorasick([np.arange(10, dtype=np.uint8)[::2]])  # not contiguous
    # iterables and buffer types are accepted
    AhoCorasick(iter(["hello", "world"]))
    AhoCorasick(p for p in ["a", "b"])
    BytesAhoCorasick([memoryview(b"hello"), bytearray(b"world")])


def test_enums_and_deprecated_constants():
    assert MATCHKIND_STANDARD == MatchKind.Standard
    assert MATCHKIND_LEFTMOST_FIRST == MatchKind.LeftmostFirst
    assert MATCHKIND_LEFTMOST_LONGEST == MatchKind.LeftmostLongest
    assert MatchKind.Standard != MatchKind.LeftmostFirst
    assert {i.name for i in Implementation} == {"NoncontiguousNFA", "ContiguousNFA", "DFA"}
    import ahocorasick_rs
    assert ahocorasick_rs.AhoCorasick is AhoCorasick and ahocorasick_rs.MATCHKIND_STANDARD == MatchKind.Standard


def test_store_patterns_heuristic():
    # reference src/lib.rs:162-184: store iff the running total of code points stays <= 4096
    assert AhoCorasick(["a" * 4096])._patterns is not None
    assert AhoCorasick(["a" * 4097])._patterns is None
    assert AhoCorasick(["a" * 4000, "b" * 97])._patterns is None
    assert AhoCorasick(["é" * 4096])._patterns is not None  # code points, not bytes
    assert AhoCorasick(["a" * 5000], store_patterns=True)._patterns is not None
    assert AhoCorasick(["a"], store_patterns=False)._patterns is None


def test_overlapping_refused_before_any_work_and_no_cpu_fallback():
    ac = AhoCorasick(["a"], matchkind=MatchKind.LeftmostFirst)
    with pytest.raises(ValueError):
        ac.find_matches_as_indexes("", overlapping=True)
    with pytest.raises(ValueError):
        BytesAhoCorasick([b"a"], matchkind=MatchKind.LeftmostLongest).find_matches_as_indexes(b"", overlapping=True)
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):  # fails loudly: no silent CPU path
            AhoCorasick(["a"]).find_matches_as_indexes("abc")


def test_many_patterns_construction():
    # reference tests/test_ac.py:86-100 exercises > 10 240 patterns (chunked ingestion)
    pats = [f"p{i}_{i * 7919 % 1000}_" for i in range(30_000)]
    ac = AhoCorasick(pats)
    assert ac._ac.n_patterns == 30_000 and ac._patterns is None


def test_scan_in_windows_against_the_oracle():
    """The window cut used for haystacks above one call's range (matcher.scan_in_windows), with the oracle as the
    per-window scanner: byte offsets and code point indexes, multi-byte characters straddling the cuts."""
    import numpy as np
    from ahocorasick_rs_b200.matcher import scan_in_windows
    from oracle import Oracle

    rng = np.random.default_rng(17)
    text = "".join(rng.choice(list("ab—é☃cd"), size=30_000))
    upats = ["a—", "—é", "☃c", "b", "é☃c", "dd", "—"]
    orc = Oracle([u.encode() for u in upats], "Standard")
    raw = np.frombuffer(text.encode(), dtype=np.uint8)
    halo = max(len(u.encode()) for u in upats) - 1

    def bytes_scan(w):
        return np.array([(0, p, s, e) for (p, s, e) in orc.find(w.tobytes(), overlapping=True)], dtype=np.int64).reshape(-1, 4)

    def cp_scan(w):
        wb = w.tobytes()
        cont = np.cumsum(np.concatenate([[0], (np.frombuffer(wb, dtype=np.uint8) & 0xC0) == 0x80]))
        return np.array([(0, p, s - cont[s], e - cont[e]) for (p, s, e) in orc.find(wb, overlapping=True)], dtype=np.int64).reshape(-1, 4)

    exp_b = orc.find(raw.tobytes(), overlapping=True)
    exp_c = orc.find_str(text, overlapping=True)
    assert len(exp_b) > 5000
    for wbytes in (halo + 1, 17, 1000, 4099, len(raw) + 5):
        got = np.concatenate(scan_in_windows(bytes_scan, raw, wbytes, halo, False))
        assert [tuple(r[1:]) for r in got.tolist()] == exp_b, wbytes
        got = np.concatenate(scan_in_windows(cp_scan, raw, wbytes, halo, True))
        assert [tuple(r[1:]) for r in got.tolist()] == exp_c, wbytes

