"""The host plumbing the batch queries share (ahocorasick_rs_b200/matcher.py): the cut of a batch into calls
(_haystack_runs), the windows of one oversized haystack (_windows) and the staging layout of host batches
(_pack_host).  CPU tensors and numpy only: no device, no library."""
import numpy as np
import pytest
import torch

from ahocorasick_rs_b200.matcher import _haystack_runs, _pack_host, _windows


def _offsets(lens):
    offs = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(np.asarray(lens, dtype=np.int64), out=offs[1:])
    return torch.from_numpy(offs)


def _check_runs(lens, limit):
    offs = _offsets(lens)
    runs = list(_haystack_runs(offs, limit))
    n = len(lens)
    h = 0
    for h0, h1, start, end, large in runs:
        assert h0 == h and h1 > h0, "the items cover [0, n) once, in order"
        assert (start, end) == (int(offs[h0]), int(offs[h1]))
        if large:
            assert h1 == h0 + 1 and lens[h0] > limit
        else:
            assert end - start <= limit
            assert all(x <= limit for x in lens[h0:h1])
            assert h1 == n or lens[h1] > limit or offs[h1 + 1] - start > limit, "a run is the longest that fits"
        h = h1
    assert h == n
    assert [r[0] for r in runs if r[4]] == [i for i, x in enumerate(lens) if x > limit]
    return runs


@pytest.mark.parametrize("seed", range(20))
def test_runs_random(seed):
    rng = np.random.default_rng(seed)
    limit = int(rng.integers(1, 64))
    n = int(rng.integers(0, 60))
    lens = [int(x) for x in rng.integers(0, 2 * limit + 2, n)]
    lens = [0 if rng.random() < 0.2 else x for x in lens]   # empty haystacks between the others
    _check_runs(lens, limit)


def test_runs_edges():
    assert _check_runs([], 10) == []
    assert _check_runs([0, 0, 0], 10) == [(0, 3, 0, 0, False)]   # a zero-byte run is yielded too
    assert _check_runs([10], 10) == [(0, 1, 0, 10, False)]       # exactly at the limit: a run
    assert _check_runs([11], 10) == [(0, 1, 0, 11, True)]        # limit + 1: oversized
    assert _check_runs([11, 12, 30], 10) == [(0, 1, 0, 11, True), (1, 2, 11, 23, True), (2, 3, 23, 53, True)]
    assert _check_runs([3, 4, 3, 0, 1], 10) == [(0, 4, 0, 10, False), (4, 5, 10, 11, False)]
    assert _check_runs([2, 11, 0, 2], 10) == [(0, 1, 0, 2, False), (1, 2, 2, 13, True), (2, 4, 13, 15, False)]
    assert list(_haystack_runs(torch.zeros(1, dtype=torch.int64), 10)) == []   # n == 0


def _check_windows(total_len, limit, halo):
    wins = list(_windows(total_len, limit, halo))
    if total_len == 0:
        assert wins == []
        return
    assert wins[0][0] == 0 and wins[-1][1] == total_len
    for w0, w1 in wins:
        assert 0 < w1 - w0 <= limit
    for (a0, a1), (b0, b1) in zip(wins, wins[1:]):
        assert a1 - b0 == halo and b1 > a1, "consecutive windows share exactly halo bytes"


@pytest.mark.parametrize("seed", range(20))
def test_windows_random(seed):
    rng = np.random.default_rng(seed)
    halo = int(rng.integers(0, 20))
    limit = halo + int(rng.integers(1, 30))
    _check_windows(int(rng.integers(0, 400)), limit, halo)


def test_windows_edges():
    assert list(_windows(10, 10, 3)) == [(0, 10)]
    assert list(_windows(11, 10, 3)) == [(0, 10), (7, 11)]
    assert list(_windows(5, 1, 0)) == [(i, i + 1) for i in range(5)]
    _check_windows(0, 10, 3)
    for limit, halo in ((3, 3), (2, 3), (0, 0)):
        with pytest.raises(ValueError):
            list(_windows(100, limit, halo))


def _check_pack(chunks):
    buf = np.full(1 << 14, 0xAB, dtype=np.uint8)
    asked = []

    def alloc(nbytes):
        asked.append(nbytes)
        return buf[:nbytes]

    offs, head, total = _pack_host(alloc, chunks)
    raw = [bytes(memoryview(c)) for c in chunks]
    n = len(chunks)
    assert asked == [head + total]
    assert head % 512 == 0 and head >= 8 * (n + 1)
    assert np.array_equal(offs, np.concatenate([[0], np.cumsum([len(r) for r in raw], dtype=np.int64)]))
    assert np.array_equal(buf[:8 * (n + 1)].view(np.int64), offs)
    assert total == sum(len(r) for r in raw) and buf[head:head + total].tobytes() == b"".join(raw)


def test_pack_host():
    rng = np.random.default_rng(7)
    blobs = [rng.integers(0, 256, k, dtype=np.uint8) for k in (0, 1, 513, 7, 0, 100)]
    for kind in (bytes, bytearray, lambda b: memoryview(bytes(b)), lambda b: b):
        chunks = [kind(b) if kind is not bytes else b.tobytes() for b in blobs]
        _check_pack(chunks)          # many
        _check_pack(chunks[2:3])     # one (no join)
        _check_pack(chunks[:1])      # one, empty
    _check_pack([])
    _check_pack([b"x"] * 70)         # the offsets pass the first 512 bytes
