"""Per-pattern biases for completing tokens on the GPU: bias_completing_tokens_ against the brute-force model
(tests/sequence_bias_model.py), bit for bit, for every id width, logits dtype and strided row views; all -inf biases
against the mask; history edge cases, ids outside the token range and match kinds; pattern sets and per-request values
through duplicates; scale; the argument checks; CUDA-graph replay; a generation loop against a torch baseline of the
sequence-bias processor; two threads."""
import threading

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import MatchKind, TokenAhoCorasick

from .completions_model import ALPHA, LIMIT, random_patterns
from .sequence_bias_model import BiasModel, apply_sums, model_bias_sums

pytestmark = pytest.mark.gpu

WIDTHS = [torch.uint16, torch.int32, torch.int64]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
SMALL = [a for a in ALPHA if a < 20000]
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


def batch(hists, dtype=torch.int64):
    flat = [x for h in hists for x in h]
    offs = np.zeros(len(hists) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hists], out=offs[1:])
    if dtype == torch.uint16:
        tokens = torch.from_numpy(np.asarray(flat, dtype=np.uint16)).cuda()
    else:
        tokens = torch.tensor(flat, dtype=dtype, device="cuda")
    return tokens, torch.from_numpy(offs).cuda()


def assert_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    g, w = got.detach().cpu().contiguous().view(BITS[got.dtype]), want.contiguous().view(BITS[want.dtype])
    bad = (g != w).nonzero()
    assert bad.numel() == 0, (bad[:5].tolist(), got.cpu()[tuple(bad[:5].T)], want[tuple(bad[:5].T)])


def rand_bias(rng, n):
    """Random float32 biases, not dyadic, over several magnitudes: any other summation order would show."""
    return (rng.standard_normal(n) * 10.0 ** rng.integers(-2, 3, n)).astype(np.float32)


def setup(seed, alphabet, n_pats=20, max_len=5, kind=MatchKind.Standard):
    rng = np.random.default_rng(seed)
    pats = random_patterns(rng, n_pats, max_len, np.array(alphabet))
    pats += [list(pats[0]), list(pats[1])]   # more duplicates
    return rng, pats, TokenAhoCorasick(pats, matchkind=kind)


def histories(rng, pats, alphabet, n=40):
    out = [[]]
    for i in range(n):
        h = [int(x) for x in rng.choice(alphabet, int(rng.integers(0, 20)))]
        if i % 2:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        out.append(h)
    return out


# ---- the model, bit for bit ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("width", WIDTHS, ids=str)
def test_bias(width, dtype):
    rng, pats, tac = setup(2, SMALL)
    hists = histories(rng, pats, SMALL)
    b = rand_bias(rng, len(pats))
    bias = torch.from_numpy(b).cuda()
    V = 20011
    logits = (torch.randn(len(hists), V, device="cuda") * 4).to(dtype)
    want = apply_sums(logits, [model_bias_sums(pats, h, b) for h in hists])
    out = tac.bias_completing_tokens_(logits, *batch(hists, width), bias)
    assert out is logits
    assert_bits(logits, want)
    assert tac.last_stats["mode"] == "completions" and tac.last_stats["entries"] == len(pats)
    # a strided row view of a 3-D tensor: scores[:, 1, :V]; the rest of the tensor is untouched
    scores = (torch.randn(len(hists), 3, V + 7, device="cuda") * 4).to(dtype)
    full = scores.clone()
    view = scores[:, 1, :V]
    assert view.stride(1) == 1 and view.stride(0) == 3 * (V + 7)
    want = apply_sums(full[:, 1, :V], [model_bias_sums(pats, h, b) for h in hists])
    tac.bias_completing_tokens_(view, *batch(hists, width), bias)
    assert_bits(scores[:, 1, :V], want)
    assert torch.equal(scores[:, 0].view(BITS[dtype]), full[:, 0].view(BITS[dtype]))
    assert torch.equal(scores[:, 2].view(BITS[dtype]), full[:, 2].view(BITS[dtype]))
    assert torch.equal(scores[:, 1, V:].view(BITS[dtype]), full[:, 1, V:].view(BITS[dtype]))


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_all_minus_inf_equals_the_mask(dtype):
    rng, pats, tac = setup(3, SMALL, n_pats=40)
    hists = histories(rng, pats, SMALL, n=60)
    logits = (torch.randn(len(hists), 20000, device="cuda") * 4).to(dtype)
    masked = tac.mask_completing_tokens_(logits.clone(), *batch(hists))
    biased = tac.bias_completing_tokens_(logits.clone(), *batch(hists), torch.full((len(pats),), float("-inf"), device="cuda"))
    assert torch.equal(biased.view(BITS[dtype]), masked.view(BITS[dtype]))


def test_order_and_ieee_edges_on_the_device():
    """The order decides the float32 sum (1e8, 1, -1e8 over three depths); a lone -0.0 keeps a -0.0 logit; +inf and
    -inf together give NaN; overflow to inf; ties by pid between duplicates."""
    pats = [[5], [3, 5], [2, 3, 5], [6], [6], [7], [7], [8]]
    tac = TokenAhoCorasick(pats)
    b = np.array([1e8, 1.0, -1e8, -0.0, -0.0, float("inf"), float("-inf"), 3e38], dtype=np.float32)
    hists = [[2, 3], [3], [], [9, 2, 3]]
    logits = torch.zeros(len(hists), 10, device="cuda")
    logits[:, 6] = -0.0
    logits[:, 8] = 3e38
    want = apply_sums(logits, [model_bias_sums(pats, h, b) for h in hists])
    tac.bias_completing_tokens_(logits, *batch(hists), torch.from_numpy(b).cuda())
    got = logits.cpu()
    nan = torch.isnan(want)   # a NaN's payload is the hardware's: compare where, then the bits of the rest
    assert torch.equal(torch.isnan(got), nan)
    assert_bits(got.masked_fill(nan, 0), want.masked_fill(nan, 0))
    assert got[0, 5].item() == 0.0 and got[1, 5].item() == 1e8 and torch.signbit(got[0, 6])   # 1 + 1e8 rounds to 1e8
    assert torch.isnan(got[:, 7]).all() and torch.isinf(got[:, 8]).all()


# ---- histories -------------------------------------------------------------------------------------------------------
def test_history_edges_and_offset_clamping():
    pats = [[1, 2, 3], [2, 4], [9], [5, 5, 5, 5], [2, 3], [9]]
    tac = TokenAhoCorasick(pats)
    b = np.array([0.5, -1.25, 2.0, 3.0, 0.75, -0.125], dtype=np.float32)
    bias = torch.from_numpy(b).cuda()
    buf = [7, 1, 2, 5, 5, 5, 2, 1, 2]
    tokens = torch.tensor(buf, dtype=torch.int64, device="cuda")

    def clamp(o):
        return min(max(o, 0), len(buf))

    for a, e in [(0, 0), (0, 3), (1, 3), (3, 6), (2, 9), (5, 100), (-4, 2), (6, 2), (50, 60), (-9, -1), (9, 9), (8, 9)]:
        ca, ce = clamp(a), clamp(e)
        h = buf[ca:ce] if ce >= ca else []
        logits = torch.randn(1, 16, device="cuda")
        want = apply_sums(logits, [model_bias_sums(pats, h, b)])
        tac.bias_completing_tokens_(logits, tokens, torch.tensor([a, e], dtype=torch.int64, device="cuda"), bias)
        assert_bits(logits, want)
    # offsets[0] > 0, many rows in one call
    logits = torch.randn(3, 16, device="cuda")
    want = apply_sums(logits, [model_bias_sums(pats, buf[x:y], b) for x, y in ((2, 3), (3, 6), (6, 9))])
    tac.bias_completing_tokens_(logits, tokens, torch.tensor([2, 3, 6, 9], dtype=torch.int64, device="cuda"), bias)
    assert_bits(logits, want)
    # no rows, and an empty id buffer
    tac.bias_completing_tokens_(torch.zeros(0, 16, device="cuda"), tokens, torch.zeros(1, dtype=torch.int64, device="cuda"), bias)
    logits = torch.zeros(2, 16, device="cuda")
    tac.bias_completing_tokens_(logits, torch.zeros(0, dtype=torch.int32, device="cuda"), torch.tensor([0, 0, 5], device="cuda"), bias)
    assert logits[:, 9].tolist() == [2.0 - 0.125] * 2 and int((logits != 0).sum()) == 2


@pytest.mark.parametrize("width", [torch.int32, torch.int64], ids=str)
def test_ids_outside_the_token_range(width):
    pats = [[1, 2, 3], [2, 4], [9], [LIMIT - 1, 6], [6]]
    tac = TokenAhoCorasick(pats)
    b = np.array([1.5, 2.5, -3.5, 4.25, 0.125], dtype=np.float32)
    big = (1 << 31) - 1 if width == torch.int32 else (1 << 40)
    hists = [[-1, 1, 2], [1, -1], [LIMIT, 2], [big], [-5, LIMIT - 1], [LIMIT - 1 - (1 << 21)],
             [-(1 << 31) if width == torch.int32 else -(1 << 62)]]
    logits = torch.zeros(len(hists), 16, dtype=torch.float16, device="cuda")
    want = apply_sums(logits, [model_bias_sums(pats, h, b) for h in hists])
    tac.bias_completing_tokens_(logits, *batch(hists, width), torch.from_numpy(b).cuda())
    assert_bits(logits, want)
    assert logits[4, 6].item() == 4.25 + 0.125


def test_long_history_reads_only_the_tail():
    pats = [[3, 1, 4, 1, 5], [9, 2, 6], [5], [1, 5]]
    tac = TokenAhoCorasick(pats)
    b = np.array([1.0, 2.0, 4.0, 8.0], dtype=np.float32)
    hists = [[7] * 100000 + [3, 1, 4, 1], [3, 1, 4] + [8] * 70000 + [9, 2], [1] * 33 + [3, 1, 4, 1]]
    logits = torch.zeros(3, 10, device="cuda")
    tac.bias_completing_tokens_(logits, *batch(hists, torch.int32), torch.from_numpy(b).cuda())
    assert logits[:, 5].tolist() == [13.0, 4.0, 13.0] and logits[1, 6].item() == 2.0


def test_match_kinds_agree():
    rng = np.random.default_rng(4)
    pats = random_patterns(rng, 30, 5, np.array(SMALL))
    hists = histories(rng, pats, SMALL)
    b = rand_bias(rng, len(pats))
    logits0 = torch.randn(len(hists), 20000, device="cuda", dtype=torch.bfloat16)
    want = apply_sums(logits0, [model_bias_sums(pats, h, b) for h in hists])
    for kind in MatchKind:
        logits = logits0.clone()
        TokenAhoCorasick(pats, matchkind=kind).bias_completing_tokens_(logits, *batch(hists), torch.from_numpy(b).cuda())
        assert_bits(logits, want)


# ---- pattern sets ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64], ids=str)
def test_pattern_sets(index_dtype):
    rng, pats, tac = setup(5, SMALL, n_pats=40)
    hists = histories(rng, pats, SMALL, n=60)
    n = len(hists)
    sets = [sorted({p for p in range(len(pats)) if rng.random() < 0.4}) for _ in range(5)] + [[], list(range(len(pats)))]
    ps = tac.pattern_sets(sets)
    idx = [int(rng.integers(0, len(sets))) for _ in range(n)]
    bad = [-1, len(sets), 1 << 20] + ([(1 << 63) - 1, -(1 << 63)] if index_dtype == torch.int64 else [(1 << 31) - 1, -(1 << 31)])
    for j, v in enumerate(bad):
        idx[3 * j + 1] = v
    set_index = torch.tensor(idx, dtype=index_dtype, device="cuda")
    b = rand_bias(rng, len(pats))
    bias = torch.from_numpy(b).cuda()
    logits = torch.randn(n, 20000, device="cuda", dtype=torch.bfloat16)
    want = apply_sums(logits, [model_bias_sums(pats, h, b, set(sets[s]) if 0 <= s < len(sets) else set())
                               for h, s in zip(hists, idx)])
    before = logits.clone()
    tac.bias_completing_tokens_(logits, *batch(hists), bias, pattern_sets=ps, set_index=set_index)
    assert_bits(logits, want)
    for j in range(len(bad)):   # an index outside [0, n_sets) biases nothing
        assert torch.equal(logits[3 * j + 1].view(torch.int16), before[3 * j + 1].view(torch.int16))
    # the "all" set equals the unfiltered call
    all_idx = torch.full((n,), len(sets) - 1, dtype=index_dtype, device="cuda")
    a = tac.bias_completing_tokens_(before.clone(), *batch(hists), bias, pattern_sets=ps, set_index=all_idx)
    u = tac.bias_completing_tokens_(before.clone(), *batch(hists), bias)
    assert torch.equal(a.view(torch.int16), u.view(torch.int16))


def test_per_request_values_through_duplicates():
    """The same sequence twice, as two pids with their own biases, each in its own request's set."""
    seqs = [[1, 2, 3], [4, 5], [6]]
    pats = seqs + seqs
    tac = TokenAhoCorasick(pats)
    ps = tac.pattern_sets([[0, 1, 2], [3, 4, 5], list(range(6))])
    bias = torch.tensor([-2.0, 1.5, -0.5, 3.0, -4.0, 0.25], device="cuda")
    hists = [[1, 2], [1, 2], [1, 2], [4], [4], [4]]
    logits = torch.zeros(6, 8, device="cuda")
    set_index = torch.tensor([0, 1, 2, 0, 1, 2], dtype=torch.int32, device="cuda")
    tac.bias_completing_tokens_(logits, *batch(hists), bias, pattern_sets=ps, set_index=set_index)
    got = logits.cpu()
    assert got[:3, 3].tolist() == [-2.0, 3.0, 1.0] and got[3:, 5].tolist() == [1.5, -4.0, -2.5]
    assert got[:, 6].tolist() == [-0.5, 0.25, -0.25] * 2


# ---- scale -----------------------------------------------------------------------------------------------------------
def test_scale():
    rng = np.random.default_rng(6)
    pats = [[int(x) for x in rng.integers(0, 50000, int(rng.integers(1, 9)))] for _ in range(10000)]
    pats += [[int(a), int(b)] for a, b in zip(rng.permutation(60000) + 70000, rng.integers(0, 50000, 40000))]
    pats += [[int(x)] for x in rng.integers(0, 50000, 300)]
    long_pat = [int(x) for x in rng.choice(SMALL, 210)]
    pats += [long_pat, long_pat[-5:], long_pat[-1:]]
    tac = TokenAhoCorasick(pats)
    model = BiasModel(pats)
    b = rand_bias(rng, len(pats))
    hists = []
    for i in range(600):
        h = [int(x) for x in rng.integers(0, 130000, int(rng.integers(0, 30)))]
        if i % 3 == 0:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        hists.append(h)
    hists += [long_pat[:-1], [1] + long_pat[:-1], long_pat[:-2], long_pat[:100], long_pat[:-1] * 2]
    sums = [model(h, b) for h in hists]
    t = long_pat[-1]
    assert all(t in s for s in sums[-5:])
    logits = torch.randn(len(hists), 130000, dtype=torch.bfloat16, device="cuda")
    want = apply_sums(logits, sums)
    tac.bias_completing_tokens_(logits, *batch(hists), torch.from_numpy(b).cuda())
    assert_bits(logits, want)
    assert tac.last_stats["nodes"] > 40000


# ---- argument checks -------------------------------------------------------------------------------------------------
def test_vocabulary_and_bias_checks():
    tac = TokenAhoCorasick([[1, 2], [5, 300], [7]])
    tokens, offsets = batch([[5], [1]])
    bias = torch.tensor([1.0, 2.0, 3.0], device="cuda")
    with pytest.raises(ValueError, match="300"):
        tac.bias_completing_tokens_(torch.zeros(2, 300, device="cuda"), tokens, offsets, bias)
    logits = torch.zeros(2, 301, device="cuda")
    tac.bias_completing_tokens_(logits, tokens, offsets, bias)
    assert logits[0, 300].item() == 2.0 and logits[0, 7].item() == 3.0 and logits[1, 2].item() == 1.0
    assert int((logits != 0).sum()) == 4
    with pytest.raises(ValueError, match="rows"):
        tac.bias_completing_tokens_(torch.zeros(3, 301, device="cuda"), tokens, offsets, bias)
    with pytest.raises(ValueError, match="stride"):
        tac.bias_completing_tokens_(torch.zeros(301, 2, device="cuda").t(), tokens, offsets, bias)
    with pytest.raises(TypeError, match="logits"):
        tac.bias_completing_tokens_(torch.zeros(2, 301, device="cuda", dtype=torch.float64), tokens, offsets, bias)
    for bad in (bias.double(), bias.half(), [1.0, 2.0, 3.0], bias.to(torch.int32)):
        with pytest.raises(TypeError, match="bias"):
            tac.bias_completing_tokens_(logits, tokens, offsets, bad)
    for bad in (bias[:2], torch.zeros(4, device="cuda"), bias.reshape(1, 3), torch.zeros(0, device="cuda")):
        with pytest.raises(ValueError, match="bias"):
            tac.bias_completing_tokens_(logits, tokens, offsets, bad)
    with pytest.raises(ValueError, match="bias lives on cpu"):
        tac.bias_completing_tokens_(logits, tokens, offsets, bias.cpu())
    # a strided bias view is taken as its values
    wide = torch.zeros(6, device="cuda")
    wide[::2] = bias
    l2 = torch.zeros(2, 301, device="cuda")
    tac.bias_completing_tokens_(l2, tokens, offsets, wide[::2])
    assert torch.equal(l2, logits)
    # no patterns: nothing to add, any vocabulary works
    empty = TokenAhoCorasick([])
    ones = torch.ones(2, 1, device="cuda")
    empty.bias_completing_tokens_(ones, tokens, offsets, torch.zeros(0, device="cuda"))
    assert torch.equal(ones, torch.ones(2, 1, device="cuda"))


# ---- CUDA graph ------------------------------------------------------------------------------------------------------
def test_cuda_graph_capture_and_replay():
    rng, pats, tac = setup(8, SMALL, n_pats=50)
    sets = [sorted({p for p in range(len(pats)) if rng.random() < 0.5}) for _ in range(4)]
    ps = tac.pattern_sets(sets)
    n, L, V = 32, 16, 20000
    ids = torch.zeros(n, L, dtype=torch.int64, device="cuda")
    offsets = torch.arange(n + 1, device="cuda") * L
    set_index = torch.zeros(n, dtype=torch.int32, device="cuda")
    bias = torch.zeros(len(pats), device="cuda")
    logits = torch.zeros(n, V, device="cuda", dtype=torch.float16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            tac.bias_completing_tokens_(logits, ids.view(-1), offsets, bias, pattern_sets=ps, set_index=set_index)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tac.bias_completing_tokens_(logits, ids.view(-1), offsets, bias, pattern_sets=ps, set_index=set_index)
    for step in range(3):
        hist = [[int(x) for x in rng.choice(SMALL, L)] for _ in range(n)]
        for i in range(0, n, 2):
            p = pats[int(rng.integers(0, len(pats)))]
            if len(p) - 1 <= L:
                hist[i] = (hist[i] + p[:-1])[-L:]
        ids.copy_(torch.tensor(hist, device="cuda"))
        si = [int(rng.integers(-1, 5)) for _ in range(n)]
        set_index.copy_(torch.tensor(si, device="cuda"))
        b = rand_bias(rng, len(pats))
        bias.copy_(torch.from_numpy(b))
        logits.copy_(torch.randn(n, V, device="cuda"))
        want = apply_sums(logits, [model_bias_sums(pats, h, b, set(sets[x]) if 0 <= x < 4 else set()) for h, x in zip(hist, si)])
        g.replay()
        torch.cuda.synchronize()
        assert_bits(logits, want)


# ---- a generation loop against a torch sequence-bias processor -------------------------------------------------------
def torch_sequence_bias(logits, ids2d, pats, bias, admit):
    """Vectorised sequence-bias baseline: per length group, the rows whose tail equals p[:-1] get bias[p] at p[-1],
    accumulated in float32 (exact here: the biases are multiples of 1/4 and small), then added once and rounded."""
    n, V = logits.shape
    acc = torch.zeros(n, V, dtype=torch.float32, device=logits.device)
    by_len = {}
    for pid, p in enumerate(pats):
        by_len.setdefault(len(p), []).append(pid)
    for ln, pids in by_len.items():
        seqs = torch.tensor([pats[i] for i in pids], dtype=torch.int64, device=logits.device)
        pid_t = torch.tensor(pids, dtype=torch.int64, device=logits.device)
        hit = admit[:, pid_t]
        if ln > 1:
            if ids2d.shape[1] < ln - 1:
                continue
            hit = hit & (ids2d[:, ids2d.shape[1] - (ln - 1):, None] == seqs[:, :ln - 1].T[None]).all(dim=1)
        r, c = hit.nonzero(as_tuple=True)
        acc.index_put_((r, seqs[c, ln - 1]), bias[pid_t[c]], accumulate=True)
    return (logits.float() + acc).to(logits.dtype)


def test_generation_loop_matches_the_torch_baseline():
    rng = np.random.default_rng(9)
    V = 400
    pats = [[int(x) for x in rng.integers(0, V, int(rng.integers(2, 5)))] for _ in range(600)]
    pats += [[int(x)] for x in rng.integers(0, V, 20)]
    pats += [[7, 7], [7, 8, 7], [7, 7], [7]]
    tac = TokenAhoCorasick(pats)
    sets = [sorted({p for p in range(len(pats)) if rng.random() < 0.5}) for _ in range(8)]
    ps = tac.pattern_sets(sets)
    member = torch.zeros(8, len(pats), dtype=torch.bool, device="cuda")
    for g, s in enumerate(sets):
        member[g, torch.tensor(s, dtype=torch.int64, device="cuda")] = True
    bias = torch.tensor(rng.integers(-32, 33, len(pats)) / 4.0, dtype=torch.float32, device="cuda")   # exact sums
    n, prompt, steps = 256, 8, 64
    set_index = torch.tensor(rng.integers(0, 8, n), dtype=torch.int64, device="cuda")
    admit = member[set_index]
    ids = torch.tensor(rng.integers(0, V, (n, prompt)), dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(9)
    for t in range(steps):
        L = ids.shape[1]
        logits = torch.randn(n, V, device="cuda", generator=gen).to(torch.bfloat16)
        want = torch_sequence_bias(logits, ids, pats, bias, admit)
        tac.bias_completing_tokens_(logits, ids.reshape(-1), torch.arange(n + 1, device="cuda") * L, bias,
                                    pattern_sets=ps, set_index=set_index)
        assert torch.equal(logits.view(torch.int16), want.view(torch.int16)), t
        nxt = torch.argmax(logits.float() + torch.empty(n, V, device="cuda").exponential_(generator=gen).log().neg(), dim=1)
        ids = torch.cat([ids, nxt[:, None]], dim=1)


# ---- threads ---------------------------------------------------------------------------------------------------------
def test_two_threads_share_one_object():
    rng, pats, tac = setup(10, SMALL, n_pats=60)
    hists = histories(rng, pats, SMALL, n=80)
    b = rand_bias(rng, len(pats))
    logits0 = torch.randn(len(hists), 20000, device="cuda")
    want = apply_sums(logits0, [model_bias_sums(pats, h, b) for h in hists])
    errors = []

    def work(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                bias = torch.from_numpy(b).cuda()
                for i in range(10):
                    logits = logits0.clone()
                    tac.bias_completing_tokens_(logits, *batch(hists, WIDTHS[(k + i) % 3]), bias)
                    torch.cuda.current_stream().synchronize()
                    assert_bits(logits, want)
        except Exception as e:   # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
