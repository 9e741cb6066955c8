"""CPU counterpart of test_gpu_table_shapes.py: every pattern set of tests/table_shapes.py gets the dense-table shape
it was built for (column mode, column count, lowest byte, the column of its edge bytes, hot rows and whether the
byte-indexed table exists) under every match kind, and the image interpreter's model of the staged walker agrees with
the oracle on a short random-byte haystack with 5 hot rows, a middle count and the full hot set."""
import pytest

from oracle import Oracle
from tests import image_interp as ii
from tests.table_shapes import CASE_IDS, CASES, LATTICE, LATTICE_BYTES, batch_of, check_shape, lattice_batch, ragged_random

KINDS = ["Standard", "LeftmostFirst", "LeftmostLongest"]


@pytest.mark.parametrize("kind", range(3), ids=KINDS)
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_shape(case, kind):
    im, desc = check_shape(case, kind)
    if case.wide:
        assert desc.rows == 127                   # 127 * 512 < 64 KiB: the trap row's u16 offset still fits
        assert check_shape(case, kind, 79)[1].rows == 79


@pytest.mark.parametrize("kind", range(3), ids=KINDS)
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_staged_model_matches_oracle(case, kind):
    im, desc = check_shape(case, kind)
    orc = Oracle(case.pats, KINDS[kind])
    data, offs = ragged_random(case, seed=5, n_haystacks=4, max_len=700, empty=0.0)
    hays = [bytes(data[offs[h]:offs[h + 1]]) for h in range(len(offs) - 1)]
    exp = [(h, p, s, e) for h, hay in enumerate(hays) for (p, s, e) in orc.find(hay)]
    assert len(exp) > 0
    for H in (5, max(5, desc.rows // 2), 4096):
        for base in (0, 63):
            assert ii.emulate_scan(im, data, offs, H=H, base_addr=base, segment_bytes=128) == exp, (H, base)
    if kind == 0:
        expo = [(h, p, s, e) for h, hay in enumerate(hays) for (p, s, e) in orc.find(hay, overlapping=True)]
        assert ii.emulate_scan(im, data, offs, overlapping=True, H=desc.rows // 2, segment_bytes=128) == expo


@pytest.mark.parametrize("case", LATTICE, ids=[c.name for c in LATTICE])
def test_staged_model_on_the_high_byte_lattice(case):
    """c0 + c1 * 64 matches after the byte c0, at every chunk offset, and after no other byte of 0x7e, 0x7f, 0x80."""
    im, desc = check_shape(case, 0)
    data, offs = lattice_batch(case, seed=7)
    vals = (0x7E, 0x7F, 0x80)
    hays = [bytes(data[offs[h]:offs[h + 1]]) for h in (LATTICE_BYTES.index(v) for v in vals)]
    data, offs = batch_of(hays)
    got = ii.emulate_scan(im, data, offs, overlapping=True, H=desc.rows, segment_bytes=1024)
    orc = Oracle(case.pats, "Standard")
    assert got == [(h, p, s, e) for h, hay in enumerate(hays) for (p, s, e) in orc.find(hay, overlapping=True)]
    c0 = case.lattice[0]
    exp = [(vals.index(c0), 257 * k, 257 * k + 65) for k in range(64)] if c0 in vals else []
    assert [(h, s, e) for (h, p, s, e) in got if p == 0] == exp
