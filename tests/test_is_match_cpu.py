"""CPU tests of is_match: acb_any_match refuses bad arguments before any CUDA call, and the public methods validate
their arguments exactly as find_matches_as_indexes does, before any device work, and have no CPU fallback."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it


def _automaton(kind=0):
    L = _capi.lib()
    pats = [b"hello", b"world"]
    offs = np.array([0, 5, 10], dtype=np.uint64)
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, 2, kind, -1, C.byref(h)) == 0
    return L, h


def _any(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, flags=FAKE, scratch=FAKE):
    return L.acb_any_match(h, sieve, data, offs, n, total, flags, scratch, None)


def test_any_match_rejects_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(flags=None), "null argument"),
            (dict(scratch=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31"),
            (dict(total=(1 << 31) + 12345), "total_bytes must be below 2^31"),
            ({}, "acb_sieve_build has not been called"),   # valid arguments, but no sieve image yet
        ]
        for kw, msg in cases:
            assert _any(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_any_match(None, FAKE, FAKE, FAKE, 1, 16, FAKE, FAKE, None) == _capi.ACB_EINVAL
        assert "null argument" in _capi.last_error()
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=["Standard", "LeftmostFirst", "LeftmostLongest"])
def test_any_match_accepts_every_match_kind(kind):
    """Past the argument checks the call needs CUDA: without a device it fails with ACB_ECUDA, never ACB_EUNSUPPORTED
    or a CPU answer.  An empty byte buffer may come with a null data pointer."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the pointers here are not device memory")
    L, h = _automaton(kind)
    try:
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        for total, data in ((16, FAKE), (0, None)):
            assert _any(L, h, data=data, total=total) == _capi.ACB_ECUDA, _capi.last_error()
    finally:
        L.acb_free(h)


def _same_error(fn_a, fn_b):
    with pytest.raises(Exception) as a:
        fn_a()
    with pytest.raises(Exception) as b:
        fn_b()
    assert type(a.value) is type(b.value) and str(a.value) == str(b.value)
    return a.value


def test_is_match_validates_like_find_matches_as_indexes():
    ac = AhoCorasick(["hello"])
    for bad in (b"hello", 12, None, ["hello"]):
        e = _same_error(lambda: ac.is_match(bad), lambda: ac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            ac.is_match_batch(["ok", bad])
    bac = BytesAhoCorasick([b"hello"])
    for bad in ("hello", 12, np.zeros((2, 2), dtype=np.uint8), np.arange(10, dtype=np.uint8)[::2]):
        e = _same_error(lambda: bac.is_match(bad), lambda: bac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            bac.is_match_batch([b"ok", bad])
    bad = np.arange(4, dtype=np.int32)   # not u8
    e = _same_error(lambda: bac.is_match(bad), lambda: bac.find_matches_as_indexes(bad))
    assert isinstance(e, BufferError)


def test_is_match_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for kind in MatchKind:
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).is_match("abc")
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).is_match_batch(["abc", "x"])
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).is_match(b"abc")
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).is_match_device(torch.zeros(3, dtype=torch.uint8),
                                                                     torch.tensor([0, 3]))
