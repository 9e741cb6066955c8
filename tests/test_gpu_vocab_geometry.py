"""Vocabulary masks on the GPU at every geometry of their kernels (csrc/vocab.cuh), bit for bit against the DFA-free
reference (tests/vocab_reference.py): the state kernel's history pieces for every id width, row tiles up to the mask
kernel's tile stride and the state kernel's row stride, candidate strides past the grid's x cap, every DFA shape of
tests/table_shapes.py, the walk branches, every kernel instance with values that round, a row offset past 2^31
elements, and the host form's device batches.  Every check compares the whole logits tensor: banned elements hold the
value as torch rounds it from float32 to the dtype, everything else (padded columns too) is unchanged.  Where a test
aims at a geometry, it asserts that the geometry was reached, from the device's SM count and the launch caps."""
import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind

from . import table_shapes as ts
from . import vocab_families as vf
from .vocab_model import VocabImage, image_bytes
from .vocab_reference import VocabReference, bits, expected_logits, row_history

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
WIDTHS = [torch.uint16, torch.int32, torch.int64]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
KINDS = [MatchKind.Standard, MatchKind.LeftmostFirst, MatchKind.LeftmostLongest]
NEG_INF = float("-inf")
# the launch geometry (csrc/vocab.cuh, vocab_*_launch in csrc/capi.cu)
ROWS_PER_TILE = 16          # kVocabRows
THREADS = 256               # kVocabThreads: candidates per block pass, 8 row-warps per state block
GRID_X, GRID_Y = 4096, 65535


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _flat(hists, dtype=torch.int64):
    offs = np.zeros(len(hists) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hists], out=offs[1:])
    flat = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists] + [np.zeros(0, dtype=np.int64)])
    npt = {torch.uint16: np.uint16, torch.int32: np.int32, torch.int64: np.int64}[dtype]
    return torch.from_numpy(flat.astype(npt)).to(DEV), torch.from_numpy(offs).to(DEV)


def _check(v, ref, hists, V, ldtype=torch.float32, tdtype=torch.int64, sets=None, idx=None, ps=None, value=NEG_INF,
           pad=0, offsets=None):
    """One mask call over rows `hists` (or, with `offsets`, rows cut from the flat histories by those offsets), checked
    bit for bit; a row whose set index lies outside [0, len(sets)) bans nothing.  -> the (n, V) ban tensor."""
    tokens, offs = _flat(hists, tdtype)
    rows = hists
    if offsets is not None:
        flat = [x for h in hists for x in h]
        rows = [row_history(flat, offsets, i) for i in range(len(offsets) - 1)]
        offs = torch.tensor(offsets, dtype=torch.int64, device=DEV)
    n = len(rows)
    admitted = None
    if sets is not None:
        admitted = [set(sets[int(s)]) if 0 <= int(s) < len(sets) else set() for s in idx]
    ban = ref.table(rows, V, admitted)
    base = torch.randn(n, V + pad, device=DEV).to(ldtype)
    before = base.clone()
    logits = base[:, :V]
    it = None if idx is None else torch.tensor(idx, dtype=torch.int32, device=DEV)
    v.mask_completing_tokens_(logits, tokens, offs, ps, it, value=value)
    assert torch.equal(bits(logits), bits(expected_logits(before[:, :V], ban, value)))
    assert torch.equal(bits(base[:, V:]), bits(before[:, V:]))
    return ban


def _host_image(v):
    """The image `v` uploads, written on the host and read by the interpreter."""
    host = np.zeros(v.image_bytes, dtype=np.uint8)
    assert v._ac._L.acb_vocab_write(v._ac._h, v._blob.ctypes.data, v._offsets.ctypes.data, v.n_vocab, host.ctypes.data,
                                    v.image_bytes) == 0
    return VocabImage(host.tobytes())


# ---- history pieces: the state kernel's backwards scan ----------------------------------------------------------------
PIECE_FAMILIES = [vf.pieces(L) for L in vf.PIECE_LENS] + [vf.dam_then_empties(), vf.one_byte()]


@pytest.mark.parametrize("tdtype", WIDTHS, ids=str)
@pytest.mark.parametrize("fam", PIECE_FAMILIES, ids=[f.name for f in PIECE_FAMILIES])
def test_history_pieces(fam, tdtype):
    v = BytesAhoCorasick(fam.patterns).vocabulary(fam.vocab)
    ref = VocabReference(fam.patterns, fam.vocab)
    V = len(fam.vocab) + 3
    ban = _check(v, ref, fam.histories, V, tdtype=tdtype)
    assert bool(ban.any())
    assert v.last_stats["max_pattern_len"] == fam.need + 1
    # the state kernel's own output, the calling thread's state buffer: the DFA state after exactly the last `need`
    # bytes.  A walk over more bytes can end in the state of a whole longest pattern instead, whose row (and so every
    # ban) equals its failure state's: only the state itself shows it.
    state = v._tls.states[DEV.index][:len(fam.histories)].cpu().tolist()
    assert state == [_host_image(v).state(h) for h in fam.histories]
    stops = [vf.read_stop(fam.vocab, h, fam.need) for h in fam.histories]
    if fam.name == "pieces-1000":
        assert max(k // 32 for k in stops) + 1 >= 32
    if fam.name.startswith("pieces-"):
        assert {(1, 0), (1, 31), (2, 0), (2, 31)} <= {(k // 32, k % 32) for k in stops}
    if fam.name == "dam-empties":
        assert bool(ban[0, fam.vocab.index(b"n")]) and bool(ban[1, fam.vocab.index(b"n")])
        assert stops[0] == 1000
    # the same rows cut by offsets that start late, decrease, go negative and run past the tokens
    lens = np.cumsum([0] + [len(h) for h in fam.histories])
    offsets = [int(x) for x in lens]
    offsets[0] = -5
    for i in range(2, len(offsets) - 1, 4):
        offsets[i] -= 40
    for i in range(3, len(offsets) - 1, 7):
        offsets[i] = offsets[i - 1] - 3
    offsets[-2], offsets[-1] = int(lens[-1]) + 10, int(lens[-1]) + 100
    _check(v, ref, fam.histories, V, ldtype=torch.bfloat16, tdtype=tdtype, offsets=offsets)


# ---- row tiles ---------------------------------------------------------------------------------------------------------
def _tile_case(D, seed=3):
    rng = np.random.default_rng(seed)
    pats, vocab = vf.stride_vocab(rng, 300)
    hists = [[int(x) for x in rng.integers(0, len(vocab), int(rng.integers(0, 5)))] for _ in range(D)]
    hists[1] = [len(vocab) + 1]
    return pats, vocab, hists


def _tiles_differ(ban_rows):
    """Every tile of two or more rows holds two neighbours (cyclically within the tile) with different ban sets, so a
    ban stored to another row of its tile changes the result."""
    n = ban_rows.shape[0]
    r = torch.arange(n, device=DEV)
    r0 = r - r % ROWS_PER_TILE
    nr = torch.clamp(n - r0, max=ROWS_PER_TILE)
    nxt = r0 + (r - r0 + 1) % nr
    diff = (ban_rows != ban_rows[nxt]).any(dim=1) | (nr == 1)
    per_tile = torch.zeros((n + ROWS_PER_TILE - 1) // ROWS_PER_TILE, dtype=torch.bool, device=DEV)
    per_tile.index_put_((r // ROWS_PER_TILE,), diff, accumulate=True)
    return bool(per_tile.all())


@pytest.mark.parametrize("n_rows", [1, 15, 16, 17, 31, 33])
def test_row_tiles(n_rows):
    pats, vocab, hists = _tile_case(37)
    ac = BytesAhoCorasick(pats)
    v, ref = ac.vocabulary(vocab), VocabReference(pats, vocab)
    rows = [hists[r % 37] for r in range(n_rows)]
    ban = _check(v, ref, rows, len(vocab) + 9, ldtype=torch.float16)
    assert n_rows == 1 or _tiles_differ(ban)
    # per-row sets, with indices outside [0, n_sets) in the middle of each tile
    sets = [list(range(0, len(pats), 2)), list(range(1, len(pats), 2)), list(range(len(pats)))]
    ps = ac.pattern_sets(sets)
    idx = [(-1, 0, 1, 2, 3)[(r * 3) % 5] if r % 16 not in (0, 15) else r % 3 for r in range(n_rows)]
    _check(v, ref, rows, len(vocab), ldtype=torch.bfloat16, sets=sets, idx=idx, ps=ps)


def test_row_grid_stride_and_tile_stride():
    """65 535 x 16 + 37 rows of 31 cycled histories, V = 48, bfloat16: past the state kernel's 32 x SMs blocks of 8
    row-warps and the mask kernel's 65 535 tiles of grid.y, with a partial last tile."""
    D = 31
    n_rows = GRID_Y * ROWS_PER_TILE + 37
    assert n_rows > 32 * _sms() * 8 and (n_rows + ROWS_PER_TILE - 1) // ROWS_PER_TILE > GRID_Y and n_rows % ROWS_PER_TILE
    rng = np.random.default_rng(5)
    alpha = b"abcdefgh"
    vocab = [bytes([b]) for b in alpha] + [vf._rand(rng, alpha, int(rng.integers(0, 4))) for _ in range(40)]
    pats = [b"abc", b"bd", b"cfe", b"dd", b"ea", b"fgh", b"gc", b"hb", b"bahg", b"eeee", b"hgfedcb"]
    hists = [[int(x) for x in rng.integers(0, len(vocab), int(rng.integers(0, 6)))] for _ in range(D)]
    v, ref = BytesAhoCorasick(pats).vocabulary(vocab), VocabReference(pats, vocab)
    V = 48
    table = ref.table(hists, V)
    assert torch.unique(table, dim=0).shape[0] >= 4
    lens = np.array([len(h) for h in hists], dtype=np.int64)
    reps = n_rows // D + 1
    cycle = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists])
    tokens = torch.from_numpy(np.tile(cycle, reps)).to(DEV)
    offs = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.tile(lens, reps)[:n_rows], out=offs[1:])
    hist_of = torch.arange(n_rows, device=DEV) % D
    ban = table[hist_of]
    assert _tiles_differ(ban)
    logits = torch.randn(n_rows, V, device=DEV, dtype=torch.bfloat16)
    want = expected_logits(logits, ban, NEG_INF)
    v.mask_completing_tokens_(logits, tokens.to(torch.int32), torch.from_numpy(offs).to(DEV))
    assert torch.equal(bits(logits), bits(want))
    del logits, want, ban, tokens
    torch.cuda.empty_cache()


# ---- candidate strides -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_vocab", [255, 256, 257])
def test_candidate_strides(n_vocab):
    rng = np.random.default_rng(n_vocab)
    pats, vocab = vf.stride_vocab(rng, n_vocab)
    ac = BytesAhoCorasick(pats)
    v, ref = ac.vocabulary(vocab), VocabReference(pats, vocab)
    hists = [[int(x) for x in rng.integers(0, n_vocab, int(rng.integers(0, 5)))] for _ in range(21)]
    sets = [list(range(0, len(pats), 2)), list(range(len(pats)))]
    ps = ac.pattern_sets(sets)
    idx = [r % 3 for r in range(21)]
    for V in (n_vocab - 1, n_vocab, n_vocab + 1, n_vocab + 256, n_vocab + 300):
        ban = _check(v, ref, hists, V, pad=3)
        assert bool(ban[:, min(V, n_vocab) - 8:].any())   # bans among the last candidates
        _check(v, ref, hists, V, ldtype=torch.float16, sets=sets, idx=idx, ps=ps, pad=5)


def test_more_candidates_than_one_grid_pass():
    """Every 1-4 byte string over 32 letters (1 082 400 entries) in a seeded shuffle: past grid.x's 4096 blocks of 256
    candidates, with bans at ids past 1 048 576."""
    alpha = bytes(range(0x41, 0x61))
    vocab = vf.all_strings(alpha, 4, seed=17)
    n = len(vocab)
    V = n + 5
    assert n == 1082400 and (V + THREADS - 1) // THREADS > GRID_X
    rng = np.random.default_rng(17)
    pats = [vf._rand(rng, alpha, k) for k in (2, 3, 3, 4, 5, 5, 6, 7, 9)]
    ac = BytesAhoCorasick(pats)
    v, ref = ac.vocabulary(vocab), VocabReference(pats, vocab)
    index = {s: t for t, s in enumerate(vocab)}
    hists = [[]]
    for i in range(20):   # ids spelling a random prefix of a pattern, after random ids and sometimes a break
        p = pats[i % len(pats)]
        k = int(rng.integers(1, len(p)))
        h = [int(x) for x in rng.integers(0, n, int(rng.integers(0, 3)))] + ([-1] if i % 5 == 0 else [])
        h += [index[p[a:a + 2]] if k - a >= 2 else index[p[a:a + 1]] for a in range(0, k, 2)]
        hists.append(h)
    ban = _check(v, ref, hists, V)
    assert bool(ban[:, GRID_X * THREADS:].any())
    sets = [[0, 2, 4, 6, 8], [1, 3, 5, 7]]
    _check(v, ref, hists, V, ldtype=torch.float16, sets=sets, idx=[r % 2 for r in range(21)], ps=ac.pattern_sets(sets))


# ---- DFA shapes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS, ids=str)
@pytest.mark.parametrize("case", ts.CASES, ids=ts.CASE_IDS)
def test_table_shapes(case, kind):
    fam = vf.shape_family(case)
    v, ref = BytesAhoCorasick(fam.patterns, matchkind=kind).vocabulary(fam.vocab), VocabReference(fam.patterns, fam.vocab)
    ldtype = DTYPES[ts.CASES.index(case) % 3]
    ban = _check(v, ref, fam.histories, len(fam.vocab) + 1, ldtype=ldtype, tdtype=WIDTHS[KINDS.index(kind)])
    assert bool(ban.any())
    assert v.last_stats["columns"] == case.n_cols
    assert (v.last_stats["extra_dfa_bytes"] > 0) == (kind != MatchKind.Standard)


def test_table_shapes_reach_both_column_extremes():
    assert {c.n_cols for c in ts.CASES} >= {2, 256}


# ---- walk branches -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS, ids=str)
@pytest.mark.parametrize("make", vf.WALKS, ids=[f.__name__ for f in vf.WALKS])
def test_walk_branches(make, kind):
    fam = make()
    ac = BytesAhoCorasick(fam.patterns, matchkind=kind)
    v, ref = ac.vocabulary(fam.vocab), VocabReference(fam.patterns, fam.vocab)
    n = len(fam.patterns)
    sets = [list(range(n)), [n - 1], [1], [0], list(range(1, n, 2)), [3], [4]]
    sets = [[p for p in s if p < n] for s in sets]
    ps = ac.pattern_sets(sets)
    rows = [h for h in fam.histories for _ in range(len(sets))]
    idx = [i % len(sets) for i in range(len(rows))]
    V = len(fam.vocab)
    ban = _check(v, ref, fam.histories, V)
    fban = _check(v, ref, rows, V, ldtype=torch.bfloat16, sets=sets, idx=idx, ps=ps)
    assert bool(ban.any()) and bool(fban.any())
    img = VocabImage(image_bytes(fam.patterns, fam.vocab))
    if make is vf.one_byte:
        assert img.lvl2 == img.n_states
    if make is vf.deep_state:
        assert max(int(img.depth[img.state(h)]) for h in fam.histories) >= 100
    if make is vf.shadowed and kind == MatchKind.LeftmostFirst:
        assert v.last_stats["extra_dfa_bytes"] > 0
        r = rows.index(fam.histories[0]) + sets.index([1])
        assert bool(fban[r, fam.vocab.index(b"abcd")])   # only pid 1 admitted: "abcd" holds it


# ---- every instance and rounding -----------------------------------------------------------------------------------------
VALUES = [NEG_INF, -0.0, float("nan"), 70000.0, 1.0 + 2.0 ** -8, 3.5 * 2.0 ** -24, 5.0]


@pytest.mark.parametrize("tdtype", WIDTHS, ids=str)
@pytest.mark.parametrize("filt", [False, True])
@pytest.mark.parametrize("ldtype", DTYPES, ids=str)
def test_every_instance_and_value(ldtype, filt, tdtype):
    """Each mask instance (logits dtype x filter) and state instance (id width) at 37 rows (3 tiles) and 600 ids (3
    blocks); values that are inf in float16, ties in bfloat16 and subnormal ties in float16, -0.0 and NaN bit for bit."""
    rng = np.random.default_rng(11)
    pats, vocab = vf.stride_vocab(rng, 600)
    ac = BytesAhoCorasick(pats)
    v, ref = ac.vocabulary(vocab), VocabReference(pats, vocab)
    hists = [[int(x) for x in rng.integers(0, len(vocab), int(rng.integers(0, 5)))] for _ in range(37)]
    sets = [list(range(0, len(pats), 2)), list(range(len(pats)))] if filt else None
    idx = [r % 3 for r in range(37)] if filt else None
    for value in VALUES:
        _check(v, ref, hists, 611, ldtype=ldtype, tdtype=tdtype, sets=sets, idx=idx, ps=ac.pattern_sets(sets) if filt else None,
               value=value, pad=2)


# ---- a row offset past 2^31 elements --------------------------------------------------------------------------------------
def test_row_offsets_past_2_31_elements():
    rng = np.random.default_rng(13)
    pats, vocab = vf.stride_vocab(rng, 64)
    v, ref = BytesAhoCorasick(pats).vocabulary(vocab), VocabReference(pats, vocab)
    stride, n, V = (1 << 27) + 5, 17, 64
    hists = [[int(x) for x in rng.integers(0, 64, int(rng.integers(0, 5)))] for _ in range(n)]
    ban = ref.table(hists, V)
    assert bool(ban[16].any()) and 16 * stride > (1 << 31)
    storage = torch.zeros(16 * stride + V, dtype=torch.bfloat16, device=DEV)
    view = torch.as_strided(storage, (n, V), (stride, 1))
    v.mask_completing_tokens_(view, *_flat(hists))
    assert torch.equal(bits(view), bits(expected_logits(torch.zeros(n, V, dtype=torch.bfloat16, device=DEV), ban, NEG_INF)))
    assert int(torch.count_nonzero(storage)) == int(ban.sum())   # nothing written outside the rows
    del view, storage
    torch.cuda.empty_cache()


# ---- the host form's device batches ----------------------------------------------------------------------------------------
def test_host_form_batches(monkeypatch):
    fam = vf.pieces(65)
    v, ref = BytesAhoCorasick(fam.patterns).vocabulary(fam.vocab), VocabReference(fam.patterns, fam.vocab)
    hists = fam.histories
    k = 7 if len(hists) % 7 else 8   # rows per device batch: several batches and an uneven last one
    monkeypatch.setattr(type(v), "ROWS_ELEMENTS", k * v.n_vocab)
    assert len(hists) > 2 * k and len(hists) % k
    pats = [[i % 2] if i % 3 else [0, 1] for i in range(len(hists))]
    assert v.completing_tokens_batch(hists, patterns=pats) == [ref(h, set(p)) for h, p in zip(hists, pats)]
    assert v.completing_tokens_batch(hists) == [ref(h) for h in hists]
