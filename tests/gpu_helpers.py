"""Helpers shared by the GPU test modules: the `kernel` fixture that forces each kernel variant in turn, and the
comparison of a device scan with the CPU oracle -- and, for code points, with the decoded text itself and, for
small inputs, with the brute-force statement of the semantics (tests/spec_bruteforce.py), so that the C oracle is
not the only reference."""
import contextlib

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, _capi
from oracle import Oracle

from .spec_bruteforce import spec_find

KINDS = [MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest]
# (kind, overlapping): every match kind, and the overlapping search (Standard only)
SEARCHES = [(k, False) for k in KINDS] + [(MatchKind.Standard, True)]
SEARCH_IDS = ["Standard", "LeftmostFirst", "LeftmostLongest", "Overlapping"]

# name -> acb_set_tuning(kernel, hot_rows, segment_bytes, table)
VARIANTS = {
    "sieve": (5, 0, 0, 0),                       # the default engine: position-parallel filter + exact verification (scan_sieve.cuh)
    "sieve-small-tasks": (5, 0, 512, 0),         # one 512-byte window per task: every boundary case at every task start
    "staged": (2, 0, 0, 0),                      # the default: compact (column-indexed) table, one segment per lane
    "plain": (1, 0, 0, 0),
    "staged-tiny-hot": (2, 5, 0, 1),             # 5 hot rows, compact table: nearly every group leaves the hot set
    "staged-small-segments": (2, 0, 128, 0),     # 128-byte segments: speculative starts and the repair pass everywhere
    "staged-compact-table": (2, 0, 0, 1),        # column-indexed table even where the byte-indexed one would do
    "staged-byte-table": (2, 0, 0, 2),           # byte-indexed table (IDP4A transitions) wherever the patterns are ASCII
    "staged-byte-table-tiny": (2, 7, 256, 2),    # byte-indexed table forced, 7 rows, 256-byte segments
    "staged-two-per-lane": (3, 0, 0, 0),         # two segments per lane (two interleaved chains)
    "staged-two-per-lane-tiny": (3, 6, 128, 1),  # ... with 6 hot rows and 128-byte segments: careful path and repair everywhere
    "global-segments": (4, 0, 0, 0),             # segment-parallel, tables in global memory / L2 (what dense automata get)
    "global-small-segments": (4, 0, 128, 0),     # ... with 128-byte segments: speculation and repair everywhere
}
SIEVE_VARIANTS = ("sieve", "sieve-small-tasks")


def is_sieve(variant):
    return variant in SIEVE_VARIANTS


def is_segmented(variant):
    """A table walker that splits haystacks into segments scanned in parallel (all but the plain kernel)."""
    return not is_sieve(variant) and variant != "plain"


def set_kernel(kernel=0, hot_rows=0, segment_bytes=0, table=0):
    _capi.set_tuning(kernel, hot_rows, segment_bytes, table)


@contextlib.contextmanager
def forced(variant):
    set_kernel(*VARIANTS[variant])
    try:
        yield variant
    finally:
        set_kernel(0)


@pytest.fixture(params=list(VARIANTS))
def kernel(request):
    with forced(request.param):
        yield request.param


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def dev_at(a, shift):
    """`a` on the device, `shift` bytes past the start of a fresh allocation: the segment and task grids are
    anchored at aligned addresses at or before the buffer, so this moves every grid line relative to the data."""
    a = np.ascontiguousarray(a)
    buf = torch.zeros(shift + len(a) + 1, dtype=torch.uint8, device="cuda")
    out = buf[shift:shift + len(a)]
    if len(a):
        out.copy_(torch.from_numpy(a))
    return out


def gpu_batch(ac, data, offs, overlapping=False, **kw):
    d = data if isinstance(data, torch.Tensor) else dev(data)
    m, moffs, total = ac.scan_device(d, dev(offs), overlapping, **kw)
    return m.cpu().numpy().view(np.uint32), moffs.cpu().numpy(), total


def make_ac(pats_bytes, kind, codepoints=False, implementation=None):
    if codepoints:
        return AhoCorasick([p.decode() for p in pats_bytes], kind, implementation=implementation)
    return BytesAhoCorasick(pats_bytes, kind, implementation=implementation)


SPEC_BYTES = 8192   # up to this size (and this many patterns) a batch is also checked against the brute-force statement
SPEC_PATTERNS = 64


def check_text(pats_bytes, kind, data, offs, m, moffs, overlapping, codepoints):
    """Checks that need no oracle.  Code points: every record slices the decoded haystack back to its pattern.
    Small inputs: the records equal the brute-force statement's, haystack by haystack."""
    data = np.asarray(data)
    small = int(offs[-1] - offs[0]) <= SPEC_BYTES and len(pats_bytes) <= SPEC_PATTERNS
    if not codepoints and not small:
        return
    pats = [p.decode() for p in pats_bytes] if codepoints else list(pats_bytes)
    for h in range(len(offs) - 1):
        a, b = int(moffs[h]), int(moffs[h + 1])
        if a == b and not small:
            continue
        raw = data[offs[h]:offs[h + 1]].tobytes()
        hay = raw.decode("utf-8") if codepoints else raw
        rows = m[a:b]
        if codepoints:
            for _, pid, s, e in rows.tolist():
                assert hay[s:e] == pats[pid], (h, pid, s, e)
        if small:
            got = [tuple(r) for r in rows[:, 1:].tolist()]
            assert got == spec_find(pats, hay, kind.name, overlapping), h


def check_batch(pats_bytes, kind, data, offs, overlapping=False, codepoints=False, implementation=None, ac=None, shift=None,
                capacity=None):
    """Scan (data, offs) on the device and compare records, per-haystack offsets and the total with the oracle bit for
    bit.  `ac`: an automaton to scan with (its last_stats then describe this scan); `shift`: place the data that many
    bytes into a fresh device allocation.  -> the total."""
    orc = Oracle(pats_bytes, kind.name)
    total, counts, rec = orc.scan_batch(data, offs, overlapping=overlapping, codepoints=codepoints)
    if ac is None:
        ac = make_ac(pats_bytes, kind, codepoints, implementation)
    d = dev_at(data, shift) if shift is not None else data
    kw = {"capacity": capacity} if capacity is not None else {}
    m, moffs, gtotal = gpu_batch(ac, d, offs, overlapping, **kw)
    assert gtotal == total
    assert moffs[0] == 0 and np.array_equal(np.diff(moffs), counts.astype(np.int64))
    assert np.array_equal(m, rec)
    check_text(pats_bytes, kind, data, offs, m, moffs, overlapping, codepoints)
    return total
