"""CPU tests of find_first: the three C entry points refuse bad arguments before any CUDA call, the public methods
validate their arguments exactly as find_matches_as_indexes does and have no CPU fallback, and the claim the
first-match kernel rests on -- a haystack's first match is the minimum of ONE packed 64-bit key per matching end
position, taken at the deepest pattern ending there -- holds against the oracle on thousands of seeded cases."""
import ctypes as C

import numpy as np
import pytest

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .spec_bruteforce import occurrences, spec_find

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
KIND_NAMES = ["Standard", "LeftmostFirst", "LeftmostLongest"]


def _automaton(kind=0):
    L = _capi.lib()
    pats = [b"hello", b"world"]
    offs = np.array([0, 5, 10], dtype=np.uint64)
    blob = np.frombuffer(b"".join(pats), dtype=np.uint8)
    h = C.c_void_p()
    assert L.acb_build(blob.ctypes.data, offs.ctypes.data, 2, kind, -1, C.byref(h)) == 0
    return L, h


def _find(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, total=16, keys=FAKE, scratch=FAKE):
    return L.acb_find_first(h, sieve, data, offs, n, total, keys, scratch, None)


def _rows(L, h, sieve=FAKE, data=FAKE, offs=FAKE, n=1, keys=FAKE, rows=FAKE):
    return L.acb_first_rows(h, sieve, data, offs, n, keys, rows, None)


def _cp(L, data=FAKE, offs=FAKE, n=1, total=16, rows=FAKE, out=FAKE + 64):
    return L.acb_rows_to_codepoints(data, offs, n, total, rows, out, None)


def test_entry_points_reject_bad_arguments_without_a_device():
    L, h = _automaton()
    try:
        launches = L.acb_launch_count()
        find_cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(keys=None), "null argument"),
            (dict(scratch=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            (dict(total=1 << 31), "total_bytes must be below 2^31"),
            (dict(total=(1 << 31) + 12345), "total_bytes must be below 2^31"),
            ({}, "acb_sieve_build has not been called"),   # valid arguments, but no sieve image yet
        ]
        for kw, msg in find_cases:
            assert _find(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_find_first(None, FAKE, FAKE, FAKE, 1, 16, FAKE, FAKE, None) == _capi.ACB_EINVAL
        assert "null argument" in _capi.last_error()
        rows_cases = [
            (dict(sieve=None), "null argument"),
            (dict(offs=None), "null argument"),
            (dict(keys=None), "null argument"),
            (dict(rows=None), "null argument"),
            (dict(n=-1), "n_haystacks out of range"),
            (dict(n=0xffffffff), "n_haystacks out of range"),
            ({}, "acb_sieve_build has not been called"),
        ]
        for kw, msg in rows_cases:
            assert _rows(L, h, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_first_rows(None, FAKE, FAKE, FAKE, 1, FAKE, FAKE, None) == _capi.ACB_EINVAL
        cp_cases = [
            (dict(offs=None), "null argument"),
            (dict(rows=None), "null argument"),
            (dict(out=None), "null argument"),
            (dict(data=None), "null argument"),
            (dict(out=FAKE), "must not be dev_rows"),
            (dict(n=-1), "n_haystacks out of range"),
        ]
        for kw, msg in cp_cases:
            kw.setdefault("rows", FAKE)
            assert _cp(L, **kw) == _capi.ACB_EINVAL, kw
            assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert L.acb_launch_count() == launches
    finally:
        L.acb_free(h)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_entry_points_accept_every_match_kind(kind):
    """Past the argument checks the calls need CUDA: without a device they fail with ACB_ECUDA, never ACB_EUNSUPPORTED
    or a CPU answer.  An empty byte buffer may come with a null data pointer."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the pointers here are not device memory")
    L, h = _automaton(kind)
    try:
        assert L.acb_sieve_build(h, 64 * 1024, 0) > 0
        for total, data in ((16, FAKE), (0, None)):
            assert _find(L, h, data=data, total=total) == _capi.ACB_ECUDA, _capi.last_error()
            assert _cp(L, data=data, total=total) == _capi.ACB_ECUDA, _capi.last_error()
        assert _rows(L, h) == _capi.ACB_ECUDA, _capi.last_error()
    finally:
        L.acb_free(h)


def _same_error(fn_a, fn_b):
    with pytest.raises(Exception) as a:
        fn_a()
    with pytest.raises(Exception) as b:
        fn_b()
    assert type(a.value) is type(b.value) and str(a.value) == str(b.value)
    return a.value


def test_find_first_validates_like_find_matches_as_indexes():
    ac = AhoCorasick(["hello"])
    for bad in (b"hello", 12, None, ["hello"]):
        e = _same_error(lambda: ac.find_first(bad), lambda: ac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            ac.find_first_batch(["ok", bad])
    bac = BytesAhoCorasick([b"hello"])
    for bad in ("hello", 12, np.zeros((2, 2), dtype=np.uint8), np.arange(10, dtype=np.uint8)[::2]):
        e = _same_error(lambda: bac.find_first(bad), lambda: bac.find_matches_as_indexes(bad))
        assert isinstance(e, TypeError)
        with pytest.raises(TypeError):
            bac.find_first_batch([b"ok", bad])
    bad = np.arange(4, dtype=np.int32)   # not u8
    e = _same_error(lambda: bac.find_first(bad), lambda: bac.find_matches_as_indexes(bad))
    assert isinstance(e, BufferError)


def test_find_first_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    for kind in MatchKind:
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).find_first("abc")
        with pytest.raises(RuntimeError):
            AhoCorasick(["a"], matchkind=kind).find_first_batch(["abc", "x"])
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).find_first(b"abc")
        with pytest.raises(RuntimeError):
            BytesAhoCorasick([b"a"], matchkind=kind).find_first_device(torch.zeros(3, dtype=torch.uint8), torch.tensor([0, 3]))


# ---------------------------------------------------------------- the key order (what the kernel computes, in Python)
def pack_key(kind, pid, start, end):
    """The u64 key of include/acb200.h (acb_find_first) for a match (pid, start, end) in bytes."""
    if kind == 0:
        return end << 32 | (0xffffffff - (end - start))
    if kind == 1:
        return start << 32 | pid
    return start << 32 | (0xffffffff - end)


def unpack_key(kind, key, pats, hay):
    """acb_first_rows in Python: (start, end) names the pattern as the lowest index with those bytes."""
    hi, lo = key >> 32, key & 0xffffffff
    if kind == 1:
        return lo, hi, hi + len(pats[lo])
    end = hi if kind == 0 else 0xffffffff - lo
    start = end - (0xffffffff - lo) if kind == 0 else hi
    return min(i for i, p in enumerate(pats) if p == hay[start:end]), start, end


def first_by_keys(kind, pats, hay, overlapping):
    """One candidate per end position -- the longest pattern ending there, lowest index among equal bytes (the deepest
    terminal node of the reverse trie) -- and the minimum of their keys."""
    deepest = {}
    for pid, s, e in overlapping:
        best = deepest.get(e)
        if best is None or s < best[1] or (s == best[1] and pid < best[0]):
            deepest[e] = (pid, s, e)
    if not deepest:
        return None
    key = min(pack_key(kind, *m) for m in deepest.values())
    return unpack_key(kind, key, pats, hay)


@pytest.mark.parametrize("kind", [0, 1, 2], ids=KIND_NAMES)
def test_key_order_picks_the_oracles_first_match(kind):
    rng = np.random.default_rng(1000 + kind)
    checked = 0
    for case in range(3000):
        alpha = b"abc" if case % 3 else b"ab"
        n_pats = int(rng.integers(1, 9))
        pats = [bytes(rng.choice(list(alpha), size=int(rng.integers(1, 6))).astype(np.uint8)) for _ in range(n_pats)]
        if case % 5 == 0:
            pats.append(pats[int(rng.integers(0, len(pats)))])   # a duplicate: ranked by index
        if case % 7 == 0:
            pats.append(pats[0] + pats[-1])                      # nested patterns
        hay = bytes(rng.choice(list(alpha), size=int(rng.integers(0, 40))).astype(np.uint8))
        oracle = Oracle(pats, kind)
        over = Oracle(pats, 0).find(hay, overlapping=True)          # every occurrence, whatever the kind
        first = oracle.find(hay)
        want = tuple(first[0]) if first else None
        assert first_by_keys(kind, pats, hay, over) == want, (pats, hay)
        if case % 10 == 0:   # the brute-force statement of the semantics agrees with the oracle
            assert sorted(over) == sorted(occurrences(pats, hay))
            spec = spec_find(pats, hay, KIND_NAMES[kind])
            assert (tuple(spec[0]) if spec else None) == want
        checked += want is not None
    assert checked > 1500


def test_kinds_differ_on_nested_and_duplicate_patterns():
    pats = [b"abcd", b"b", b"bcd", b"ab", b"abcd", b"abcdef"]
    hay = b"xxabcdefxx"
    over = Oracle(pats, 0).find(hay, overlapping=True)
    got = [first_by_keys(k, pats, hay, over) for k in range(3)]
    assert got == [(3, 2, 4), (0, 2, 6), (5, 2, 8)]
    assert got == [tuple(Oracle(pats, k).find(hay)[0]) for k in range(3)]
