"""CPU tests of the token-id format (include/acb200.h, csrc/tokens.cuh): acb_tokens_encode_host against an independent
numpy statement of the format for every id width, the edge ids and the first-bad-index report; both entry points refuse
bad arguments before any CUDA call; TokenAhoCorasick validates patterns and arguments before any device work; and the
little-endian counterexample that the format's marker bit exists for."""
import ctypes as C

import numpy as np
import pytest

import ahocorasick_rs
from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, TokenAhoCorasick, _capi
from oracle import Oracle

from .spec_bruteforce import spec_find

FAKE = 1 << 20   # a non-null "device pointer": the argument checks must not dereference it
NO_BAD = (1 << 64) - 1
EDGE_IDS = [0, 127, 128, (1 << 14) - 1, 1 << 14, (1 << 21) - 1]
WIDTHS = {2: np.uint16, 4: np.int32, 8: np.int64}


def numpy_format(ids):
    """The format stated again, independently of the library: 0x80 | t >> 14, (t >> 7) & 0x7f, t & 0x7f per id."""
    t = np.asarray(ids, dtype=np.int64)
    out = np.empty((len(t), 3), dtype=np.uint8)
    out[:, 0] = 0x80 | (t >> 14)
    out[:, 1] = (t >> 7) & 0x7F
    out[:, 2] = t & 0x7F
    return out.reshape(-1)


def host_encode(ids, token_bytes):
    a = np.ascontiguousarray(ids, dtype=WIDTHS[token_bytes])
    out = np.full(3 * len(a) + 1, 0xEE, dtype=np.uint8)   # one guard byte past the end
    bad = np.full(1, NO_BAD, dtype=np.uint64)
    rc = _capi.lib().acb_tokens_encode_host(a.ctypes.data if len(a) else None, token_bytes, len(a),
                                            out.ctypes.data, bad.ctypes.data)
    assert rc == _capi.ACB_OK, _capi.last_error()
    assert out[-1] == 0xEE
    return out[:-1], int(bad[0])


@pytest.mark.parametrize("token_bytes", [2, 4, 8])
def test_host_encode_matches_numpy_statement(token_bytes):
    rng = np.random.default_rng(token_bytes)
    hi = 1 << 16 if token_bytes == 2 else 1 << 21
    edges = [t for t in EDGE_IDS if t < hi] + [hi - 1]
    for n in list(range(0, 20)) + [67, 1000]:
        ids = rng.integers(0, hi, n)
        if n:
            ids[rng.integers(0, n, min(n, 4))] = rng.choice(edges, min(n, 4))
        got, bad = host_encode(ids, token_bytes)
        assert bad == NO_BAD
        assert np.array_equal(got, numpy_format(ids))
    got, bad = host_encode(edges, token_bytes)
    assert bad == NO_BAD and np.array_equal(got, numpy_format(edges))


def test_format_marks_only_first_bytes():
    got, _ = host_encode(np.arange(0, 1 << 21, 997), 4)
    assert np.all((got[0::3] & 0x80) == 0x80) and np.all((got[1::3] & 0x80) == 0) and np.all((got[2::3] & 0x80) == 0)


def test_empty_input():
    got, bad = host_encode([], 4)
    assert got.size == 0 and bad == NO_BAD
    L = _capi.lib()
    bad = np.full(1, NO_BAD, dtype=np.uint64)
    assert L.acb_tokens_encode_host(None, 8, 0, None, bad.ctypes.data) == _capi.ACB_OK and bad[0] == NO_BAD


@pytest.mark.parametrize("token_bytes,value", [(4, -1), (8, -1), (4, 1 << 21), (8, 1 << 21), (8, (1 << 62) + 5), (8, -(1 << 63))])
def test_host_encode_reports_first_bad_index(token_bytes, value):
    ids = np.arange(40) % 1000
    ids_t = np.asarray(ids, dtype=WIDTHS[token_bytes])
    ids_t[17] = value
    ids_t[30] = value
    _, bad = host_encode(ids_t, token_bytes)
    assert bad == 17
    # the caller's preset is a lower bound: an earlier report stays
    a = np.ascontiguousarray(ids_t)
    out = np.empty(3 * len(a), dtype=np.uint8)
    b = np.full(1, 5, dtype=np.uint64)
    assert _capi.lib().acb_tokens_encode_host(a.ctypes.data, token_bytes, len(a), out.ctypes.data, b.ctypes.data) == _capi.ACB_OK
    assert b[0] == 5


def test_entry_points_refuse_bad_arguments():
    L = _capi.lib()
    bad = np.full(1, NO_BAD, dtype=np.uint64)
    for tb in (0, 1, 3, 16):
        assert L.acb_tokens_encode_host(FAKE, tb, 4, FAKE, bad.ctypes.data) == _capi.ACB_EINVAL
        assert L.acb_tokens_encode(FAKE, tb, 4, FAKE, FAKE, None) == _capi.ACB_EINVAL
    assert "token_bytes" in _capi.last_error()
    assert L.acb_tokens_encode_host(None, 4, 4, FAKE, bad.ctypes.data) == _capi.ACB_EINVAL
    assert L.acb_tokens_encode_host(FAKE, 4, 4, None, bad.ctypes.data) == _capi.ACB_EINVAL
    assert L.acb_tokens_encode_host(FAKE, 4, 4, FAKE, None) == _capi.ACB_EINVAL
    assert L.acb_tokens_encode(None, 4, 4, FAKE, FAKE, None) == _capi.ACB_EINVAL
    assert L.acb_tokens_encode(FAKE, 4, 4, FAKE, None, None) == _capi.ACB_EINVAL
    assert L.acb_tokens_encode(FAKE, 4, 1 << 60, FAKE, FAKE, None) == _capi.ACB_EINVAL
    assert "n_tokens" in _capi.last_error()


def test_little_endian_ids_match_inside_tokens_and_the_format_does_not():
    """Pattern [1], haystack [256, 0]: as little-endian int32 the pattern's bytes 01 00 00 00 occur at byte 1, inside
    token 0; in the format they cannot, because only a token's first byte has the high bit set."""
    le_pat, le_hay = np.array([1], np.int32).tobytes(), np.array([256, 0], np.int32).tobytes()
    assert Oracle([le_pat]).find(le_hay) == [(0, 1, 5)]
    assert spec_find([le_pat], le_hay) == [(0, 1, 5)]
    fmt_pat, fmt_hay = numpy_format([1]).tobytes(), numpy_format([256, 0]).tobytes()
    assert Oracle([fmt_pat]).find(fmt_hay) == [] and spec_find([fmt_pat], fmt_hay) == []
    for kind in ("Standard", "LeftmostFirst", "LeftmostLongest"):
        assert spec_find([fmt_pat], numpy_format([0, 1, 256, 1]).tobytes(), kind) == [(0, 3, 6), (0, 9, 12)]


def test_pattern_validation():
    with pytest.raises(ValueError, match="You passed in an empty pattern"):
        TokenAhoCorasick([[1, 2], []])
    with pytest.raises(ValueError, match="You passed in an empty pattern"):
        TokenAhoCorasick([np.zeros(0, dtype=np.uint16)])
    with pytest.raises(TypeError):
        TokenAhoCorasick([[1, 2.5]])
    with pytest.raises(TypeError):
        TokenAhoCorasick([["a"]])
    with pytest.raises(TypeError):
        TokenAhoCorasick([[True, False]])
    with pytest.raises(TypeError):
        TokenAhoCorasick([[[1, 2], [3, 4]]])
    with pytest.raises(TypeError):
        TokenAhoCorasick([5])
    with pytest.raises(TypeError):
        TokenAhoCorasick(5)
    for value in (-1, 1 << 21, 1 << 70):
        with pytest.raises(ValueError, match=rf"pattern 1: token 2 = {value} is outside"):
            TokenAhoCorasick([[1], [3, 4, value]])
    with pytest.raises(ValueError, match=r"pattern 0: token 1 = 18446744073709551615"):
        TokenAhoCorasick([np.array([3, (1 << 64) - 1], dtype=np.uint64)])
    with pytest.raises(TypeError):
        TokenAhoCorasick([[1]], matchkind="Standard")
    with pytest.raises(TypeError):
        TokenAhoCorasick([[1]], implementation=2)


def test_pattern_inputs_of_every_kind_build_the_same_automaton():
    torch = pytest.importorskip("torch")
    seqs = [[464, 3290], (17,), np.array([5, 6, 7], np.uint16), np.array([8], np.int32), np.array([9, (1 << 21) - 1], np.int64),
            np.array([10], np.uint8), torch.tensor([11, 12], dtype=torch.int64), torch.tensor([13], dtype=torch.int32)]
    ac = TokenAhoCorasick(seqs, MatchKind.LeftmostLongest)
    assert ac.max_pattern_len == 9
    assert ac._ac.n_patterns == len(seqs) and ac._ac.matchkind == MatchKind.LeftmostLongest
    assert ahocorasick_rs.TokenAhoCorasick is TokenAhoCorasick


def test_overlapping_leftmost_refused_before_device_work():
    ac = TokenAhoCorasick([[1, 2], [2]], MatchKind.LeftmostFirst)
    for call in (lambda: ac.find_matches_as_indexes([1, 2], overlapping=True),
                 lambda: ac.count_matches([1, 2], overlapping=True),
                 lambda: ac.count_matches_by_pattern_batch([[1, 2]], overlapping=True),
                 lambda: ac.matching_patterns([1, 2], overlapping=True),
                 lambda: ac.stream(overlapping=True),
                 lambda: ac.stream_batch(4, overlapping=True),
                 lambda: ac.count_matches_stream(overlapping=True),
                 lambda: ac.count_matches_stream_batch(4, overlapping=True)):
        with pytest.raises(ValueError, match="does not support overlapping"):
            call()


def test_host_forms_validate_haystacks_before_device_work():
    ac = TokenAhoCorasick([[1, 2]])
    with pytest.raises(ValueError, match=r"haystack 1: token 0 = -3 is outside"):
        ac.is_match_batch([[1, 2], [-3]])
    with pytest.raises(TypeError):
        ac.find_matches_as_indexes(b"\x01\x02")
    with pytest.raises(TypeError):
        ac.count_matches("12")
    with pytest.raises(TypeError):
        ac.find_first([1.0, 2.0])


def test_stream_seam_limit_is_stated_in_tokens():
    ac = TokenAhoCorasick([list(range(1000))])
    n = ac._ac.WINDOW_BYTES // (2 * (3 * 1000 - 1)) + 1
    with pytest.raises(ValueError, match=r"streams x 2 x \(3 x 1000 - 1\).*1000 tokens"):
        ac.stream_batch(n)
    with pytest.raises(ValueError, match="1000 tokens"):
        ac.find_first_stream_batch(n)
    ac.stream_batch(n - 1)   # (no device work until the first feed)
    with pytest.raises(TypeError):
        ac.stream_batch(2.0)
