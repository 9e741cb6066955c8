"""GPU tests (-m gpu) of the table walkers on every dense-table shape the builder makes.

The staged walker is compiled once per column layout (range, class, byte-indexed), and the builder picks the layout
from the bytes the patterns use; the kernel variants only force the kernel and its knobs.  Each pattern set of
tests/table_shapes.py is aimed at one layout edge -- one column, lo = 0, hi = 0xff, 256 range columns with the unused
byte in the "other" column on either side, both sides of the 5/4 rule, 255 and 256 used bytes, the byte-indexed
table at its 0x7e edge and ruled out by 0x7f -- and asserts that shape on the host before it runs.  Every variant and
search then runs it on ragged batches of random bytes (shifted 0, 1 and 63 bytes off the copy grid), on the
high-byte lattice, and for ASCII sets on UTF-8 text through the str class, against the oracle bit for bit.  Each run
also asserts which layout ran.  The 256-column sets also run with a hot-table budget large enough that the 16-bit
row-offset cap binds (127 rows, of which the launch takes 119 through the prefix copy)."""
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from ahocorasick_rs_b200 import matcher  # noqa: E402

from .gpu_helpers import SEARCH_IDS, SEARCHES, VARIANTS, check_batch, kernel, make_ac  # noqa: E402,F401 (kernel: the fixture)
from .table_shapes import (ASCII, CASE_IDS, CASES, RANGE, WIDE, batch_of, check_shape, lattice_batch,  # noqa: E402
                           ragged_random, utf8_texts)

WIDE_IDS = [c.name for c in WIDE]
ASCII_IDS = [c.name for c in ASCII]
BIG_BUDGET = 1 << 20   # hot-table bytes: with 256 columns, hot_rows_for's 16-bit cap (127 rows) binds first


def layout_ran(variant, ac, im):
    """The layout of the walker that answered the last scan, from the forced tuning, the image header and
    last_stats: sieve, plain, global (kernel 4: tables in global memory), ascii (the byte-indexed table), or the
    compact table's column mode."""
    kern, _, _, table = VARIANTS[variant]
    st = ac._ac.last_stats
    if st["engine"] == "sieve":
        return "sieve"
    if kern == 1:
        return "plain"
    if kern == 4 or (kern == 0 and st["global_table"]):
        assert st["groups"] == 0   # the staged walker counts its 16-byte groups; kernel 4 does not
        return "global"
    assert st["groups"] > 0
    if kern == 2 and table == 2 and st["hot_rows128"] > 0:
        return "ascii"
    return "range" if im.col_mode == RANGE else "class"


def expected_layout(variant, case):
    kern, _, _, table = VARIANTS[variant]
    if kern == 5:
        return "sieve"
    if kern == 1:
        return "plain"
    if kern == 4:
        return "global"
    if kern == 2 and table == 2 and case.byte_table:
        return "ascii"
    return "range" if case.mode == RANGE else "class"


def check_stats(variant, case, ac, im, max_rows):
    assert layout_ran(variant, ac, im) == expected_layout(variant, case)
    st = ac._ac.last_stats
    if st["engine"] == "table":
        assert st["hot_rows"] == min(max_rows, im.n_states - 1, 65535 // (2 * im.n_cols))
        assert (st["hot_rows128"] > 0) == case.byte_table
        assert st["hot_rows128"] == (min(st["hot_rows"], 255) if case.byte_table else 0)
    return st


def run_case(case, kind, overlapping, variant, seed):
    ac = make_ac(case.pats, kind)
    max_rows = ac._ac._max_hot_rows()   # the rows the host asks the image for, from HOT_TABLE_BYTES
    im, _ = check_shape(case, kind.value, max_rows)
    data, offs = ragged_random(case, seed)
    traps = 0
    for shift in (0, 1, 63):
        assert check_batch(case.pats, kind, data, offs, overlapping, ac=ac, shift=shift) > 0
        st = check_stats(variant, case, ac, im, max_rows)
        traps += st.get("traps", 0)
    # a small batch: also checked against the brute-force statement (sets of at most 64 patterns)
    data, offs = ragged_random(case, seed + 1, n_haystacks=12, max_len=400)
    check_batch(case.pats, kind, data, offs, overlapping, ac=ac)
    check_stats(variant, case, ac, im, max_rows)
    if case.lattice:
        data, offs = lattice_batch(case, seed + 2)
        assert check_batch(case.pats, kind, data, offs, overlapping, ac=ac, shift=0) > 0
        check_stats(variant, case, ac, im, max_rows)
    return max_rows, traps, st


@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_table_shape_random_bytes(case, kind, overlapping, kernel):
    max_rows, traps, st = run_case(case, kind, overlapping, kernel, seed=31)
    if case.wide:
        assert max_rows == 79          # HOT_TABLE_BYTES // 512 - 1: the launch takes the whole image in one bulk copy
        if st["engine"] == "table":
            assert st["hot_rows"] == 79
        if kernel == "staged":
            assert traps > 0


@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("case", WIDE, ids=WIDE_IDS)
def test_wide_rows_at_the_offset_cap(case, kind, overlapping, kernel, monkeypatch):
    """256 columns with a 1 MiB hot-table budget: the image gets 127 rows (the trap row must start below 64 KiB of u16
    offsets) and the staged launch keeps 119 of them (its table stays below 60 KiB), so it copies a prefix."""
    monkeypatch.setattr(matcher._Automaton, "HOT_TABLE_BYTES", BIG_BUDGET)
    max_rows, traps, st = run_case(case, kind, overlapping, kernel, seed=47)
    assert max_rows == BIG_BUDGET // 512 - 1
    if st["engine"] == "table":
        assert st["hot_rows"] == 127
    if kernel == "staged":
        assert traps > 0


@pytest.mark.parametrize("kind,overlapping", SEARCHES, ids=SEARCH_IDS)
@pytest.mark.parametrize("case", ASCII, ids=ASCII_IDS)
def test_table_shape_code_points(case, kind, overlapping, kernel):
    """ASCII pattern sets through the str class on UTF-8 text with 1- to 4-byte characters, each character's last
    byte at every chunk offset in front of the lattice run: the byte-indexed table with code points folds every byte of
    a multi-byte character onto its "other" column."""
    im, _ = check_shape(case, kind.value)
    texts = utf8_texts(case, seed=53)
    data, offs = batch_of([t.encode() for t in texts])
    ac = make_ac(case.pats, kind, codepoints=True)
    for shift in (0, 1):
        check_batch(case.pats, kind, data, offs, overlapping, codepoints=True, ac=ac, shift=shift)
        assert layout_ran(kernel, ac, im) == expected_layout(kernel, case)
