"""Completing tokens on the GPU: the CSR, the logits mask and the host forms against the brute-force model
(tests/completions_model.py) for every id width and logits dtype, history edge cases and the offset clamping rule,
match kinds, pattern sets, scale, the vocabulary check, CUDA-graph capture, a generation loop and two threads."""
import threading

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import MatchKind, TokenAhoCorasick

from .completions_model import ALPHA, LIMIT, CompletionModel, model_completing, random_patterns

pytestmark = pytest.mark.gpu

WIDTHS = [torch.uint16, torch.int32, torch.int64]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
SMALL = [a for a in ALPHA if a < 20000]   # edge ids that fit a small vocabulary (and uint16)
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


def csr_lists(ids, ro):
    ids, ro = ids.cpu().tolist(), ro.cpu().tolist()
    return [ids[ro[i]:ro[i + 1]] for i in range(len(ro) - 1)]


def check_mask(before, after, want, value=float("-inf")):
    """Rows of `after` hold `value` exactly at the ids of `want`, and are bit-identical to `before` everywhere else."""
    n, V = before.shape
    ban = torch.zeros(n, V, dtype=torch.bool, device=before.device)
    for i, ts in enumerate(want):
        if ts:
            ban[i, torch.tensor(ts, device=before.device)] = True
    bits = BITS[before.dtype]
    assert torch.equal(after.view(bits)[~ban], before.view(bits)[~ban])
    fill = torch.full((1,), value, dtype=before.dtype, device=before.device)
    assert torch.equal(after[ban], fill.expand(int(ban.sum())))


def setup(seed, alphabet, n_pats=20, max_len=5, kind=MatchKind.Standard):
    rng = np.random.default_rng(seed)
    pats = random_patterns(rng, n_pats, max_len, np.array(alphabet))
    return rng, pats, TokenAhoCorasick(pats, matchkind=kind)


def histories(rng, pats, alphabet, n=40):
    out = [[]]
    for i in range(n):
        h = [int(x) for x in rng.choice(alphabet, int(rng.integers(0, 20)))]
        if i % 2:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        out.append(h)
    return out


# ---- the forms against the model -------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", WIDTHS, ids=str)
def test_csr_and_host_forms(width):
    alphabet = [a for a in ALPHA if width != torch.uint16 or a < 65536]
    rng, pats, tac = setup(1, alphabet)
    hists = histories(rng, pats, alphabet)
    want = [model_completing(pats, h) for h in hists]
    ids, ro = tac.completing_tokens_device(*batch(hists, width))
    assert ids.dtype == torch.int64 and ro.dtype == torch.int64 and ro.shape == (len(hists) + 1,)
    assert csr_lists(ids, ro) == want
    assert tac.last_stats["mode"] == "completions" and tac.last_stats["entries"] == len(pats)
    assert tac.completing_tokens_batch(hists) == want
    assert tac.completing_tokens(hists[3]) == want[3]
    np_hist = np.asarray(hists[5], dtype=np.int64)
    assert tac.completing_tokens(np_hist) == want[5]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("width", WIDTHS, ids=str)
def test_mask(width, dtype):
    rng, pats, tac = setup(2, SMALL)
    hists = histories(rng, pats, SMALL)
    want = [model_completing(pats, h) for h in hists]
    V = 20011
    logits = torch.randn(len(hists), V, device="cuda").to(dtype)
    before = logits.clone()
    out = tac.mask_completing_tokens_(logits, *batch(hists, width))
    assert out is logits
    check_mask(before, logits, want)
    # a strided row view of a 3-D tensor: scores[:, 1, :V]
    scores = torch.randn(len(hists), 3, V + 7, device="cuda").to(dtype)
    full = scores.clone()
    view = scores[:, 1, :V]
    assert view.stride(1) == 1 and view.stride(0) == 3 * (V + 7)
    tac.mask_completing_tokens_(view, *batch(hists, width), value=-7.0)
    check_mask(full[:, 1, :V], scores[:, 1, :V], want, value=-7.0)
    assert torch.equal(scores[:, 0].view(BITS[dtype]), full[:, 0].view(BITS[dtype]))
    assert torch.equal(scores[:, 2].view(BITS[dtype]), full[:, 2].view(BITS[dtype]))
    assert torch.equal(scores[:, 1, V:].view(BITS[dtype]), full[:, 1, V:].view(BITS[dtype]))


def test_input_ids_reshape():
    rng, pats, tac = setup(3, SMALL)
    n, L = 16, 12
    ids = torch.tensor(rng.choice(SMALL, (n, L)), dtype=torch.int64, device="cuda")
    ids[::2, L - len(pats[0]) + 1:] = torch.tensor(pats[0][:-1], device="cuda") if len(pats[0]) > 1 else ids[::2, L:]
    logits = torch.zeros(n, 20000, device="cuda")
    tac.mask_completing_tokens_(logits, ids.reshape(-1), torch.arange(n + 1, device="cuda") * L)
    want = [model_completing(pats, r) for r in ids.tolist()]
    check_mask(torch.zeros_like(logits), logits, want)


# ---- histories -------------------------------------------------------------------------------------------------------
def test_history_edges_and_offset_clamping():
    pats = [[1, 2, 3], [2, 4], [9], [5, 5, 5, 5]]
    tac = TokenAhoCorasick(pats)
    buf = [7, 1, 2, 5, 5, 5, 2, 1, 2]
    tokens = torch.tensor(buf, dtype=torch.int64, device="cuda")
    n_tok = len(buf)

    def clamp(o):
        return min(max(o, 0), n_tok)

    offs = [(0, 0), (0, 3), (1, 3), (3, 6), (2, 9), (5, 100), (-4, 2), (6, 2), (50, 60), (-9, -1), (9, 9), (8, 9)]
    starts = torch.tensor([a for a, _ in offs], dtype=torch.int64, device="cuda")
    ends = torch.tensor([b for _, b in offs], dtype=torch.int64, device="cuda")
    want = []
    for a, b in offs:
        a, b = clamp(a), clamp(b)
        want.append(model_completing(pats, buf[a:b] if b >= a else []))
    # rows as consecutive offsets: row i = [o[i], o[i + 1]), so build each pair as its own 2-entry call
    for i, (a, b) in enumerate(offs):
        o = torch.stack([starts[i], ends[i]])
        ids, ro = tac.completing_tokens_device(tokens, o)
        assert csr_lists(ids, ro) == [want[i]], (a, b)
        logits = torch.zeros(1, 16, device="cuda")
        tac.mask_completing_tokens_(logits, tokens, o)
        check_mask(torch.zeros_like(logits), logits, [want[i]])
    # offsets[0] > 0 and many rows in one call
    o = torch.tensor([2, 3, 6, 9], dtype=torch.int64, device="cuda")
    assert csr_lists(*tac.completing_tokens_device(tokens, o)) == [model_completing(pats, buf[2:3]),
                                                                    model_completing(pats, buf[3:6]),
                                                                    model_completing(pats, buf[6:9])]
    # no rows
    ids, ro = tac.completing_tokens_device(tokens, torch.zeros(1, dtype=torch.int64, device="cuda"))
    assert ids.numel() == 0 and ro.tolist() == [0]
    tac.mask_completing_tokens_(torch.zeros(0, 16, device="cuda"), tokens, torch.zeros(1, dtype=torch.int64, device="cuda"))
    # an empty token buffer
    empty = torch.zeros(0, dtype=torch.int32, device="cuda")
    assert csr_lists(*tac.completing_tokens_device(empty, torch.tensor([0, 0, 5], device="cuda"))) == [[9], [9]]


@pytest.mark.parametrize("width", [torch.int32, torch.int64], ids=str)
def test_ids_outside_the_token_range(width):
    pats = [[1, 2, 3], [2, 4], [9], [LIMIT - 1, 6]]
    tac = TokenAhoCorasick(pats)
    big = (1 << 31) - 1 if width == torch.int32 else (1 << 40)
    hists = [[-1, 1, 2], [1, -1], [LIMIT, 2], [big], [-5, LIMIT - 1], [LIMIT - 1 - (1 << 21)], [-(1 << 31) if width == torch.int32 else -(1 << 62)]]
    want = [model_completing(pats, h) for h in hists]
    assert want[0] == [3, 4, 9] and want[1] == [9] and want[4] == [6, 9]
    assert csr_lists(*tac.completing_tokens_device(*batch(hists, width))) == want
    logits = torch.zeros(len(hists), LIMIT, dtype=torch.float16, device="cuda")
    tac.mask_completing_tokens_(logits, *batch(hists, width))
    check_mask(torch.zeros_like(logits), logits, want)


def test_long_history_reads_only_the_tail():
    pats = [[3, 1, 4, 1, 5], [9, 2, 6], [5]]
    tac = TokenAhoCorasick(pats)
    hists = [[7] * 100000 + [3, 1, 4, 1], [3, 1, 4] + [8] * 70000 + [9, 2], [1] * 33 + [3, 1, 4, 1]]
    want = [model_completing(pats, h) for h in hists]
    assert want == [[5], [5, 6], [5]]
    assert csr_lists(*tac.completing_tokens_device(*batch(hists, torch.int32))) == want
    assert tac.completing_tokens_batch(hists) == want


# ---- match kinds -----------------------------------------------------------------------------------------------------
def test_match_kinds_agree():
    rng = np.random.default_rng(4)
    pats = random_patterns(rng, 30, 5, np.array(SMALL))
    hists = histories(rng, pats, SMALL)
    got = []
    for kind in MatchKind:
        tac = TokenAhoCorasick(pats, matchkind=kind)
        lists = csr_lists(*tac.completing_tokens_device(*batch(hists)))
        logits = torch.zeros(len(hists), 20000, device="cuda")
        tac.mask_completing_tokens_(logits, *batch(hists))
        got.append((lists, logits, tac.completing_tokens_batch(hists)))
    for lists, logits, host in got[1:]:
        assert lists == got[0][0] and torch.equal(logits, got[0][1]) and host == got[0][2]
    assert got[0][0] == [model_completing(pats, h) for h in hists]


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
    for j, b in enumerate(bad):
        idx[3 * j + 1] = b
    set_index = torch.tensor(idx, dtype=index_dtype, device="cuda")
    want = [model_completing(pats, h, set(sets[s]) if 0 <= s < len(sets) else set()) for h, s in zip(hists, idx)]
    tokens, offsets = batch(hists)
    assert csr_lists(*tac.completing_tokens_device(tokens, offsets, pattern_sets=ps, set_index=set_index)) == want
    logits = torch.randn(n, 20000, device="cuda", dtype=torch.bfloat16)
    before = logits.clone()
    tac.mask_completing_tokens_(logits, tokens, offsets, pattern_sets=ps, set_index=set_index)
    check_mask(before, logits, want)
    # the "all" set equals the unfiltered call; host forms take patterns= per history
    all_idx = torch.full((n,), len(sets) - 1, dtype=index_dtype, device="cuda")
    assert csr_lists(*tac.completing_tokens_device(tokens, offsets, pattern_sets=ps, set_index=all_idx)) == \
        csr_lists(*tac.completing_tokens_device(tokens, offsets))
    host_sets = [sets[s] if 0 <= s < len(sets) else [] for s in idx]
    assert tac.completing_tokens_batch(hists, patterns=host_sets) == want
    assert tac.completing_tokens(hists[1], patterns=sets[0]) == model_completing(pats, hists[1], set(sets[0]))


# ---- scale -----------------------------------------------------------------------------------------------------------
def test_scale():
    rng = np.random.default_rng(6)
    pats = [[int(x) for x in rng.integers(0, 50000, int(rng.integers(1, 9)))] for _ in range(10000)]
    pats += [[int(a), int(b)] for a, b in zip(rng.permutation(60000) + 70000, rng.integers(0, 50000, 40000))]
    long_pat = [int(x) for x in rng.choice(SMALL, 210)]
    pats.append(long_pat)
    tac = TokenAhoCorasick(pats)
    model = CompletionModel(pats)
    hists = []
    for i in range(600):
        h = [int(x) for x in rng.integers(0, 130000, int(rng.integers(0, 30)))]
        if i % 3 == 0:
            h += pats[int(rng.integers(0, len(pats)))][:-1]
        hists.append(h)
    hists += [long_pat[:-1], [1] + long_pat[:-1], long_pat[:-2], long_pat[:100], long_pat[:-1] * 2]
    want = [model(h) for h in hists]
    assert all(long_pat[-1] in w for w in (want[-5], want[-4], want[-1]))
    ids, ro = tac.completing_tokens_device(*batch(hists))
    assert csr_lists(ids, ro) == want
    assert tac.last_stats["entries"] == len(pats) and tac.last_stats["nodes"] > 40000
    logits = torch.zeros(len(hists), 130000, dtype=torch.bfloat16, device="cuda")
    tac.mask_completing_tokens_(logits, *batch(hists))
    check_mask(torch.zeros_like(logits), logits, want)


# ---- the vocabulary check --------------------------------------------------------------------------------------------
def test_vocabulary_check():
    tac = TokenAhoCorasick([[1, 2], [5, 300], [7]])
    tokens, offsets = batch([[5], [1]])
    with pytest.raises(ValueError, match="300"):
        tac.mask_completing_tokens_(torch.zeros(2, 300, device="cuda"), tokens, offsets)
    logits = torch.zeros(2, 301, device="cuda")
    tac.mask_completing_tokens_(logits, tokens, offsets)
    check_mask(torch.zeros_like(logits), logits, [[7, 300], [2, 7]])
    with pytest.raises(ValueError, match="rows"):
        tac.mask_completing_tokens_(torch.zeros(3, 301, device="cuda"), tokens, offsets)
    with pytest.raises(ValueError, match="stride"):
        tac.mask_completing_tokens_(torch.zeros(301, 2, device="cuda").t(), tokens, offsets)
    with pytest.raises(TypeError, match="logits"):
        tac.mask_completing_tokens_(torch.zeros(2, 301, device="cuda", dtype=torch.float64), tokens, offsets)
    # no patterns: nothing is banned, any vocabulary works
    empty = TokenAhoCorasick([])
    logits = torch.ones(2, 1, device="cuda")
    empty.mask_completing_tokens_(logits, tokens, offsets)
    assert torch.equal(logits, torch.ones(2, 1, device="cuda"))
    assert empty.completing_tokens_batch([[1], []]) == [[], []]


# ---- CUDA graph ------------------------------------------------------------------------------------------------------
def test_cuda_graph_capture_and_replay():
    rng, pats, tac = setup(8, SMALL, n_pats=50)
    sets = [sorted({p for p in range(len(pats)) if rng.random() < 0.5}) for _ in range(4)]
    ps = tac.pattern_sets(sets)
    n, L, V = 32, 16, 20000
    ids = torch.zeros(n, L, dtype=torch.int64, device="cuda")
    offsets = torch.arange(n + 1, device="cuda") * L
    set_index = torch.zeros(n, dtype=torch.int32, device="cuda")
    logits = torch.zeros(n, V, device="cuda", dtype=torch.float16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            tac.mask_completing_tokens_(logits, ids.view(-1), offsets, pattern_sets=ps, set_index=set_index)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tac.mask_completing_tokens_(logits, ids.view(-1), offsets, pattern_sets=ps, set_index=set_index)
    for step in range(3):
        hist = [[int(x) for x in rng.choice(SMALL, L - 4)] + (pats[int(rng.integers(0, len(pats)))][:-1] + [0] * 4)[:4] for _ in range(n)]
        for i in range(0, n, 3):
            p = pats[int(rng.integers(0, len(pats)))]
            if len(p) - 1 <= L:
                hist[i] = (hist[i] + p[:-1])[-L:]
        ids.copy_(torch.tensor(hist, device="cuda"))
        set_index.copy_(torch.tensor([int(rng.integers(-1, 5)) for _ in range(n)], device="cuda"))
        logits.copy_(torch.randn(n, V, device="cuda"))
        before = logits.clone()
        g.replay()
        torch.cuda.synchronize()
        eager = before.clone()
        tac.mask_completing_tokens_(eager, ids.view(-1), offsets, pattern_sets=ps, set_index=set_index)
        assert torch.equal(logits.view(torch.int16), eager.view(torch.int16))
        si = set_index.tolist()
        want = [model_completing(pats, h, set(sets[s]) if 0 <= s < 4 else set()) for h, s in zip(hist, si)]
        check_mask(before, logits, want)


# ---- a generation loop -----------------------------------------------------------------------------------------------
def test_generation_loop_never_emits_a_banned_sequence():
    rng = np.random.default_rng(9)
    V = 400
    pats = [[int(x) for x in rng.integers(0, V, int(rng.integers(2, 5)))] for _ in range(600)]
    pats += [[int(x)] for x in rng.integers(0, V, 20)]
    pats += [[7, 7], [7, 8, 7]]
    tac = TokenAhoCorasick(pats)
    sets = [sorted({p for p in range(len(pats)) if rng.random() < 0.5}) for _ in range(8)]
    ps = tac.pattern_sets(sets)
    n, prompt, steps = 256, 8, 64
    set_index = torch.tensor(rng.integers(0, 8, n), dtype=torch.int64, device="cuda")
    ids = torch.tensor(rng.integers(0, V, (n, prompt)), dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(9)
    for t in range(steps):
        L = ids.shape[1]
        logits = torch.randn(n, V, device="cuda", generator=gen)
        logits[:, 7] += 3.0   # make the banned 7 7 / 7 8 7 tempting
        tac.mask_completing_tokens_(logits, ids.reshape(-1), torch.arange(n + 1, device="cuda") * L, pattern_sets=ps, set_index=set_index)
        assert bool(torch.isfinite(logits).any(dim=1).all())
        nxt = torch.argmax(logits + torch.empty_like(logits).exponential_(generator=gen).log().neg(), dim=1)
        ids = torch.cat([ids, nxt[:, None]], dim=1)
    rows = ids.cpu().tolist()
    si = set_index.cpu().tolist()
    found = tac.find_matches_as_indexes_batch(rows, overlapping=True, patterns=[sets[s] for s in si])
    for i, ms in enumerate(found):
        assert all(e <= prompt for _, _, e in ms), (i, [m for m in ms if m[2] > prompt][:3])


# ---- threads ---------------------------------------------------------------------------------------------------------
def test_two_threads_share_one_object():
    rng, pats, tac = setup(10, SMALL, n_pats=60)
    hists = histories(rng, pats, SMALL, n=80)
    want = [model_completing(pats, h) for h in hists]
    errors = []

    def work(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(10):
                    assert csr_lists(*tac.completing_tokens_device(*batch(hists, WIDTHS[k % 3]))) == want
                    logits = torch.zeros(len(hists), 20000, device="cuda")
                    tac.mask_completing_tokens_(logits, *batch(hists, WIDTHS[(k + 1) % 3]))
                    torch.cuda.current_stream().synchronize()
                    check_mask(torch.zeros_like(logits), logits, want)
                    assert tac.completing_tokens_batch(hists[:5]) == want[:5]
        except Exception as e:   # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
