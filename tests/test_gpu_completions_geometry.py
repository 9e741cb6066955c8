"""The token-id logits processors (csrc/completions.cuh) at the geometry their launches and searches change at: more
rows than one grid of 32 x SMs blocks of 8 row-warps (count, emit, mask and bias), compl_child's 32-ary search at every
fan-out where its step changes, and nodes with more than 32 entries (several ballot chunks), against CompletionModel
and the sequence-bias model."""
import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import TokenAhoCorasick

from .completions_model import CompletionModel, random_patterns
from .sequence_bias_model import BiasModel

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
WARPS_PER_BLOCK = 8   # kComplThreads / 32


def _bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32)


def _flat(hists):
    offs = np.zeros(len(hists) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hists], out=offs[1:])
    flat = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists] + [np.zeros(0, dtype=np.int64)])
    return torch.from_numpy(flat).to(DEV), torch.from_numpy(offs).to(DEV)


def _csr_equals(ids, ro, want_lists):
    counts = np.array([len(w) for w in want_lists], dtype=np.int64)
    want_ro = np.zeros(len(want_lists) + 1, dtype=np.int64)
    np.cumsum(counts, out=want_ro[1:])
    want_ids = np.concatenate([np.asarray(w, dtype=np.int64) for w in want_lists] + [np.zeros(0, dtype=np.int64)])
    return np.array_equal(ro.cpu().numpy(), want_ro) and np.array_equal(ids.cpu().numpy(), want_ids)


def test_row_grid_stride_every_mode():
    """3 x 32 x SMs x 8 + 5 rows cycled from 97 distinct histories: every warp of the grid takes three or four rows."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_rows = 3 * 32 * sms * WARPS_PER_BLOCK + 5
    D = 97
    rng = np.random.default_rng(21)
    alphabet = np.arange(0, 60)
    pats = random_patterns(rng, 40, 5, alphabet)
    tac = TokenAhoCorasick(pats)
    hists = []
    for i in range(D):
        h = [int(x) for x in rng.choice(alphabet, int(rng.integers(0, 8)))]
        if i % 2:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        hists.append(h)
    model = CompletionModel(pats)
    want = [model(h) for h in hists]
    assert len({tuple(w) for w in want}) >= 10   # rows of one warp's turns ban different ids
    hist_of = np.arange(n_rows) % D
    lens = np.array([len(h) for h in hists], dtype=np.int64)
    cycle = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists])
    reps = n_rows // D + 1
    tokens = torch.from_numpy(np.tile(cycle, reps)).to(DEV)
    offs = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.tile(lens, reps)[:n_rows], out=offs[1:])
    offs = torch.from_numpy(offs).to(DEV)
    # count and emit
    ids, ro = tac.completing_tokens_device(tokens, offs)
    assert _csr_equals(ids, ro, [want[d] for d in hist_of])
    # mask
    V = 64
    ban = torch.zeros(D, V, dtype=torch.bool, device=DEV)
    for d, w in enumerate(want):
        if w:
            ban[d, torch.tensor(w, device=DEV)] = True
    h_dev = torch.from_numpy(hist_of).to(DEV)
    logits = torch.randn(n_rows, V, device=DEV).to(torch.bfloat16)
    before = logits.clone()
    tac.mask_completing_tokens_(logits, tokens, offs, value=-3.0)
    fill = torch.tensor([-3.0], device=DEV).to(torch.bfloat16)
    assert torch.equal(_bits(logits), _bits(torch.where(ban[h_dev], fill, before)))
    # bias: per distinct history, the float32 sum of its terms; the row gets round(float(logit) + s) once
    bias = rng.standard_normal(len(pats)).astype(np.float32)
    bmodel = BiasModel(pats)
    add = torch.zeros(D, V, dtype=torch.float32, device=DEV)
    has = torch.zeros(D, V, dtype=torch.bool, device=DEV)
    for d, h in enumerate(hists):
        for t, s in bmodel(h, bias).items():
            add[d, t] = float(s)
            has[d, t] = True
    assert torch.equal(has, ban)
    logits = torch.randn(n_rows, V, device=DEV).to(torch.float16)
    before = logits.clone()
    tac.bias_completing_tokens_(logits, tokens, offs, torch.from_numpy(bias).to(DEV))
    want_l = torch.where(has[h_dev], (before.float() + add[h_dev]).to(torch.float16), before)
    assert torch.equal(_bits(logits), _bits(want_l))


FANOUTS = [1, 31, 32, 33, 1023, 1024, 1025, 32769]


def _queries(kids):
    """Every child, the tokens between children, below the first and above the last."""
    q = set(kids) | {k + 1 for k in kids} | {k - 1 for k in kids} | {0, kids[-1] + 7}
    return sorted(x for x in q if x >= 0)


@pytest.mark.parametrize("n_kids", FANOUTS)
def test_child_search_at_every_fanout(n_kids):
    """A root with n_kids children (tokens 3i + 5, each ending pattern [kid, i]): every child (so every sample point
    lane x step of every level of the search), the tokens between, below and above them."""
    kids = [3 * i + 5 for i in range(n_kids)]
    pats = [[k, i] for i, k in enumerate(kids)]
    tac = TokenAhoCorasick(pats)
    model = CompletionModel(pats)
    hists = [[q] for q in _queries(kids)] + [[kids[-1], kids[0]], [kids[0], kids[-1]], []]
    ids, ro = tac.completing_tokens_device(*_flat(hists))
    assert _csr_equals(ids, ro, [model(h) for h in hists])
    assert sum(1 for h in hists if model(h)) >= n_kids


def test_child_search_below_the_root():
    """A node below the root (token 999) with 40 children, beside root children of its own."""
    kids = [7 * i + 2 for i in range(40)]
    pats = [[k, 999, 10000 + i] for i, k in enumerate(kids)] + [[k, 20000 + i] for i, k in enumerate(kids[:5])] + [[999, 5]]
    tac = TokenAhoCorasick(pats)
    model = CompletionModel(pats)
    hists = [[q, 999] for q in _queries(kids)] + [[q] for q in _queries(kids)] + [[999], [1, 2, 999]]
    ids, ro = tac.completing_tokens_device(*_flat(hists))
    want = [model(h) for h in hists]
    assert _csr_equals(ids, ro, want)
    assert sum(1 for w in want if len(w) == 2) >= 40   # 10000 + i and 5 after every child


@pytest.mark.parametrize("n_entries", [33, 64, 65])
def test_nodes_with_many_entries(n_entries):
    """n_entries patterns ending at one node (after [11, 12]) and at the root: the count and emit ballots run over
    several 32-entry chunks; duplicates of a last token across the two nodes count once."""
    last = [100 + 3 * i for i in range(n_entries)]
    pats = [[11, 12, t] for t in last] + [[t] for t in last[::2]] + [[12, t] for t in last[1::3]]
    tac = TokenAhoCorasick(pats)
    model = CompletionModel(pats)
    hists = [[11, 12], [12], [], [11], [5, 11, 12], [12, 12]]
    ids, ro = tac.completing_tokens_device(*_flat(hists))
    want = [model(h) for h in hists]
    assert _csr_equals(ids, ro, want) and len(want[0]) == n_entries
    V = last[-1] + 3
    logits = torch.randn(len(hists), V, device=DEV)
    before = logits.clone()
    tac.mask_completing_tokens_(logits, *_flat(hists))
    ban = torch.zeros(len(hists), V, dtype=torch.bool, device=DEV)
    for i, w in enumerate(want):
        ban[i, torch.tensor(w, dtype=torch.int64, device=DEV)] = True
    assert torch.equal(_bits(logits), _bits(torch.where(ban, torch.full_like(logits, float("-inf")), before)))
    sets = [list(range(0, len(pats), 2))]
    ids, ro = tac.completing_tokens_device(*_flat(hists), tac.pattern_sets(sets), torch.zeros(len(hists), dtype=torch.int32, device=DEV))
    assert _csr_equals(ids, ro, [CompletionModel(pats, set(sets[0]))(h) for h in hists])
