"""Vocabulary masks on the GPU: TokenVocabulary.mask_completing_tokens_ bit for bit against the brute force over the
oracle (every id width, logits dtype and strided view; V above and below n_vocab; history, offset and break edges;
AhoCorasick with non-ASCII patterns), at scale against a second GPU path (the batched overlapping scan of T + vocab[t]),
with pattern sets, under CUDA-graph replay, in a generation loop, and from two threads."""
import threading

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, workloads as W

from .vocab_model import BruteModel, decoded_tail

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
PATS = [b"damn", b"\nUser:", b"ab", b"bca", b"aaaa", b"\xc3\xa9t\xc3\xa9"]
VOCAB = [b"d", b"am", b"n", b"damn", b"\n", b"User", b":", b"hello", b"", b"a", b"b", b"c", b"ab", b"xxbcaxx", b"\xc3", b"\xa9t",
         b"\xc3\xa9", b"t", b"aa", b""]


def _flat(hists, dtype=torch.int64):
    offs = np.zeros(len(hists) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hists], out=offs[1:])
    npt = {torch.uint16: np.uint16, torch.int32: np.int32, torch.int64: np.int64}[dtype]
    flat = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists] + [np.zeros(0, dtype=np.int64)]).astype(npt)
    return torch.from_numpy(flat).to(DEV), torch.from_numpy(offs).to(DEV)


def _histories(rng, n_vocab, n):
    out = [[], [-1], [n_vocab], [0, 1], [4, 5], [4, -1, 5], [14], [9, 9, 9], [12, 11], [19, 8, 0, 8, 1]]
    for i in range(n):
        h = [int(x) for x in rng.integers(0, n_vocab, int(rng.integers(0, 10)))]
        if i % 3 == 0 and h:
            h.insert(int(rng.integers(0, len(h) + 1)), int(rng.choice([-1, -7, n_vocab, n_vocab + 100, 1 << 20])))
        out.append(h)
    return out


def _bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32)


def _check(logits, before, want_rows, value):
    """Banned positions hold `value` in the logits dtype; every other element is bit-identical to `before`."""
    exp = before.clone()
    for i, ids in enumerate(want_rows):
        if ids:
            exp[i, torch.tensor(ids, device=DEV)] = value
    assert torch.equal(_bits(logits), _bits(exp))


@pytest.mark.parametrize("tdtype", [torch.uint16, torch.int32, torch.int64])
@pytest.mark.parametrize("ldtype", [torch.float32, torch.float16, torch.bfloat16])
def test_exact_mask_every_width_and_dtype(tdtype, ldtype):
    rng = np.random.default_rng(1)
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteModel(PATS, VOCAB)
    hists = _histories(rng, len(VOCAB), 40)
    if tdtype == torch.uint16:   # no negative ids: breaks are ids >= n_vocab
        hists = [[x if 0 <= x < 65536 else 60000 for x in h] for h in hists]
    tokens, offs = _flat(hists, tdtype)
    for V, strided in ((len(VOCAB), False), (len(VOCAB) + 13, True), (7, False), (1, True)):
        base = torch.randn(len(hists), V + 5 if strided else V, device=DEV).to(ldtype)
        logits = base[:, :V] if strided else base
        before = base.clone()
        v.mask_completing_tokens_(logits, tokens, offs)
        want = [brute(h, V=V) for h in hists]
        if strided:   # the columns past V are bit-identical
            assert torch.equal(base[:, V:], before[:, V:])
        _check(logits, before[:, :V], want, float("-inf"))
        assert v.last_stats["mode"] == "vocab_completions" and v.last_stats["n_vocab"] == len(VOCAB)


def test_padded_columns_are_never_written():
    v = BytesAhoCorasick([b"a"]).vocabulary([b"a", b"b", b"ba"])
    logits = torch.zeros(2, 8, device=DEV)
    tokens, offs = _flat([[1], []])
    v.mask_completing_tokens_(logits, tokens, offs, value=5.0)
    assert logits.tolist() == [[5, 0, 5, 0, 0, 0, 0, 0]] * 2


def test_offset_edges():
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteModel(PATS, VOCAB)
    flat = [7, 0, 1, 4, 5, 4, -1, 5]
    tokens = torch.tensor(flat, device=DEV)
    cases = [(1, 3), (3, 5), (5, 8), (4, 2), (-5, 2), (6, 100), (8, 8), (0, 0), (100, 200)]
    for a, b in cases:   # offsets[0] > 0, decreasing, negative and clamped offsets
        o = torch.tensor([a, b], device=DEV)
        logits = torch.zeros(1, len(VOCAB), device=DEV)
        v.mask_completing_tokens_(logits, tokens, o)
        ca, cb = (min(max(x, 0), len(flat)) for x in (a, b))
        h = flat[ca:cb] if cb >= ca else []
        assert torch.isinf(logits[0]).nonzero().flatten().tolist() == brute(h), (a, b)


def test_ac_with_non_ascii_patterns():
    pats = ["été", "naïve", "日本語"]
    vocab = [b"\xc3", b"\xa9", b"t", b"na", b"\xc3\xaf", b"ve", "日".encode(), "本".encode(), "語".encode()[:2], "語".encode()[2:], b" "]
    v = AhoCorasick(pats).vocabulary(vocab)
    brute = BruteModel([p.encode() for p in pats], vocab)
    hists = [[0, 1, 2, 0], [3, 4], [6, 7, 8], [6, 7], [0, 1, 2, 10, 0]]
    tokens, offs = _flat(hists)
    logits = torch.zeros(len(hists), len(vocab), device=DEV, dtype=torch.bfloat16)
    v.mask_completing_tokens_(logits, tokens, offs)
    got = [torch.isinf(r).nonzero().flatten().tolist() for r in logits]
    assert got == [brute(h) for h in hists]
    assert got[0] == [1] and got[2] == [9]
    assert v.completing_tokens_batch(hists) == got


@pytest.mark.parametrize("kind", list(MatchKind))
def test_host_forms_and_match_kinds(kind):
    w = BytesAhoCorasick([b"damn", b"\nUser:"], matchkind=kind).vocabulary(VOCAB[:8])   # the README's example
    assert w.completing_tokens([0, 1]) == [2, 3]
    assert w.completing_tokens([4, 5]) == [3, 6]
    assert w.completing_tokens([4, -1, 5]) == [3]
    assert w.completing_tokens(np.array([4, 5], dtype=np.uint16)) == [3, 6]
    assert (w.last_stats["extra_dfa_bytes"] == 0) == (kind == MatchKind.Standard)
    v = BytesAhoCorasick(PATS, matchkind=kind).vocabulary(VOCAB)
    rng = np.random.default_rng(5)
    hists = _histories(rng, len(VOCAB), 30) + [[10 ** 12, 0, 1]]
    brute = BruteModel(PATS, VOCAB)
    assert v.completing_tokens_batch(hists) == [brute(h) for h in hists]
    assert v.completing_tokens_batch(hists, patterns=[[0, 2]] * len(hists)) == [brute(h, {0, 2}) for h in hists]


@pytest.mark.parametrize("ldtype", [torch.float32, torch.float16, torch.bfloat16])
def test_pattern_sets(ldtype):
    rng = np.random.default_rng(9)
    ac = BytesAhoCorasick(PATS)
    v = ac.vocabulary(VOCAB)
    brute = BruteModel(PATS, VOCAB)
    sets = [[0], [1, 2], [], list(range(len(PATS))), [3, 4, 5]]
    ps = ac.pattern_sets(sets)
    hists = _histories(rng, len(VOCAB), 30)
    tokens, offs = _flat(hists)
    for idt in (torch.int32, torch.int64):
        idx = torch.tensor(rng.integers(-2, len(sets) + 2, len(hists)), dtype=idt, device=DEV)
        logits = torch.zeros(len(hists), len(VOCAB), device=DEV, dtype=ldtype)
        v.mask_completing_tokens_(logits, tokens, offs, ps, idx)
        for i, h in enumerate(hists):
            s = int(idx[i])
            want = brute(h, set(sets[s])) if 0 <= s < len(sets) else []
            assert torch.isinf(logits[i]).nonzero().flatten().tolist() == want, (i, s)
    # the "all" set equals no filter
    all_idx = torch.full((len(hists),), 3, dtype=torch.int32, device=DEV)
    a, b = torch.zeros(len(hists), 30, device=DEV, dtype=ldtype), torch.zeros(len(hists), 30, device=DEV, dtype=ldtype)
    v.mask_completing_tokens_(a, tokens, offs, ps, all_idx)
    v.mask_completing_tokens_(b, tokens, offs)
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="pattern_sets"):
        v.mask_completing_tokens_(a, tokens, offs, BytesAhoCorasick(PATS).pattern_sets(sets), all_idx)


def test_argument_errors():
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    tokens, offs = _flat([[0, 1]])
    with pytest.raises(TypeError, match="logits"):
        v.mask_completing_tokens_(torch.zeros(1, 4, device=DEV, dtype=torch.float64), tokens, offs)
    with pytest.raises(ValueError, match="rows"):
        v.mask_completing_tokens_(torch.zeros(2, 4, device=DEV), tokens, offs)
    with pytest.raises(ValueError, match="contiguous"):
        v.mask_completing_tokens_(torch.zeros(1, 8, device=DEV)[:, ::2], tokens, offs)


def _scale_case():
    """10 000 patterns from the names (each name, " " + name, name + " "), and a 128 256-entry vocabulary: the 256
    single bytes, then seeded substrings of 2-8 bytes of a text made of the haystack template and the names."""
    names = W.patterns_long()
    pats = names + [" " + n for n in names] + [n + " " for n in names]
    pats = [p.encode() for p in pats[:10000]]
    rng = np.random.default_rng(11)
    text = (W.haystack_template() + " ".join(names[int(i)] for i in rng.integers(0, len(names), 20000))).encode()
    vocab = [bytes([b]) for b in range(256)]
    for k, a in zip(rng.integers(2, 9, 128256 - 256), rng.integers(0, len(text) - 8, 128256 - 256)):
        vocab.append(text[int(a):int(a) + int(k)])
    return pats, vocab, text, rng


def _scan_reference(ac, vocab, T: bytes, admitted=None):
    """The second GPU path: every T + vocab[t] as one batch through scan_device(overlapping=True); the ids with a match
    ending past len(T) (of a pattern in `admitted`, when given)."""
    lens = np.array([len(v) for v in vocab], dtype=np.int64) + len(T)
    offs = np.zeros(len(vocab) + 1, dtype=np.int64)
    np.cumsum(lens, out=offs[1:])
    data = np.frombuffer(b"".join(T + v for v in vocab), dtype=np.uint8)
    m, _, _ = ac.scan_device(torch.from_numpy(data.copy()).to(DEV), torch.from_numpy(offs).to(DEV), overlapping=True)
    m = m.to(torch.int64)
    m = m[m[:, 3] > len(T)]
    if admitted is not None:
        keep = torch.zeros(ac._ac.n_patterns, dtype=torch.bool, device=DEV)
        keep[torch.tensor(sorted(admitted), dtype=torch.int64, device=DEV)] = True
        m = m[keep[m[:, 1]]]
    return torch.unique(m[:, 0]).tolist()


def test_scale_against_the_batched_scan():
    pats, vocab, text, rng = _scale_case()
    ac = BytesAhoCorasick(pats)
    v = ac.vocabulary(vocab)
    index = {s: t for t, s in enumerate(vocab)}
    hists = []
    for i in range(16):
        a = int(rng.integers(0, len(text) - 200))
        h, p = [], a
        while p < a + int(rng.integers(0, 120)):   # a greedy tokenization of a slice of the text
            k = next(k for k in range(8, 0, -1) if text[p:p + k] in index)
            h.append(index[text[p:p + k]])
            p += k
        if i % 4 == 3:
            h.append(-1)
        hists.append(h)
    tokens, offs = _flat(hists, torch.int32)
    logits = torch.zeros(len(hists), len(vocab), device=DEV, dtype=torch.bfloat16)
    v.mask_completing_tokens_(logits, tokens, offs)
    assert v.last_stats["tail_hit_ids"] > 0
    for i in (0, 1, 5, 7, 10, 15):
        T = decoded_tail(vocab, hists[i])[-64:]   # more than max_pattern_len - 1 bytes: all that can matter
        want = _scan_reference(ac, vocab, T)
        got = torch.isinf(logits[i].float()).nonzero().flatten().tolist()
        assert got == want, i


def test_scale_with_pattern_sets_every_logits_dtype():
    """10 000 patterns of 3-20 bytes cut from the text, in 16 sets, over the 128 256-entry vocabulary: every row of every
    logits dtype equals the batched scan filtered by the row's set.  (A miscompiled store once sent a few 16-bit bans of
    exactly this workload to another row of the tile: DESIGN §4.18.)"""
    _, vocab, text, rng = _scale_case()
    pats = []
    for k, a in zip(rng.integers(3, 21, 10000), rng.integers(0, len(text) - 20, 10000)):
        pats.append(text[int(a):int(a) + int(k)])
    ac = BytesAhoCorasick(pats)
    v = ac.vocabulary(vocab)
    sets = [[p for p in range(len(pats)) if rng.random() < 0.5] for _ in range(16)]
    ps = ac.pattern_sets(sets)
    n = 64
    ids = rng.integers(256, len(vocab), (n, 128))
    for i in range(0, n, 2):   # the first bytes of a pattern, one byte per id
        p = pats[int(rng.integers(0, len(pats)))][:-1]
        ids[i, 128 - len(p):] = list(p)
    tokens = torch.tensor(ids.reshape(-1), device=DEV)
    offs = torch.arange(n + 1, device=DEV) * 128
    idx = torch.tensor(rng.integers(0, 16, n), dtype=torch.int32, device=DEV)
    got = {}
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        logits = torch.randn(n, len(vocab), device=DEV).to(dt)
        v.mask_completing_tokens_(logits, tokens, offs, ps, idx)
        got[dt] = torch.isinf(logits.float())
    for i in range(n):
        T = decoded_tail(vocab, ids[i].tolist())[-64:]
        want = torch.zeros(len(vocab), dtype=torch.bool, device=DEV)
        hit = _scan_reference(ac, vocab, T, set(sets[int(idx[i])]))
        if hit:
            want[torch.tensor(hit, device=DEV)] = True
        for dt, g in got.items():
            assert torch.equal(g[i], want), (i, dt)


@pytest.mark.parametrize("ldtype", [torch.float32, torch.float16, torch.bfloat16])
def test_cuda_graph_replay(ldtype):
    """Capture after a warm call, replay after rewriting histories and set indices in place; a second graph for a larger
    batch (which grows the state buffer) leaves the first one valid."""
    rng = np.random.default_rng(4)
    ac = BytesAhoCorasick(PATS)
    v = ac.vocabulary(VOCAB)
    brute = BruteModel(PATS, VOCAB)
    sets = [[0, 1], list(range(len(PATS)))]
    ps = ac.pattern_sets(sets)
    L = 6
    graphs = []
    for n in (8, 40):   # the second batch is larger: its warm call replaces the state buffer
        ids = torch.zeros(n, L, dtype=torch.int64, device=DEV)
        idx = torch.zeros(n, dtype=torch.int32, device=DEV)
        offs = torch.arange(n + 1, device=DEV) * L
        logits = torch.zeros(n, len(VOCAB), device=DEV, dtype=ldtype)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            v.mask_completing_tokens_(logits, ids.reshape(-1), offs, ps, idx)   # warm: the image and the state buffer
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            v.mask_completing_tokens_(logits, ids.reshape(-1), offs, ps, idx)
        graphs.append((g, ids, idx, logits, offs))   # a graph reads its inputs in place: keep every one alive
    torch.cuda.synchronize()
    # small allocations made now would take the first buffer's memory if it had been freed; no replay may write them
    junk = [torch.full((8,), 7, dtype=torch.int32, device=DEV) for _ in range(16)]
    for _ in range(3):
        for g, ids, idx, logits, _ in graphs:
            n = ids.shape[0]
            hist = rng.integers(-1, len(VOCAB), (n, L))
            sidx = rng.integers(0, 2, n)
            ids.copy_(torch.from_numpy(hist))
            idx.copy_(torch.from_numpy(sidx))
            logits.zero_()
            g.replay()
            torch.cuda.synchronize()
            for i in range(n):
                assert torch.isinf(logits[i]).nonzero().flatten().tolist() == brute(hist[i].tolist(), set(sets[sidx[i]])), i
    assert all(bool((j == 7).all()) for j in junk)


def test_generation_loop():
    """64 rows x 64 steps of argmax after the mask: no sampled token ever ends a pattern in the text after the prompt."""
    pats = [b"damn", b"\nUser:", b"ab", b"bca", b"aaaa", b"cc"]
    ac = BytesAhoCorasick(pats)
    vocab = VOCAB + [b"cc", b"c\n", b"Us", b"er:", b"dam"]
    v = ac.vocabulary(vocab)
    n, steps, P = 64, 64, 3
    g = torch.Generator(device=DEV).manual_seed(0)
    ids = torch.randint(0, len(vocab), (n, P + steps), device=DEV, generator=g)
    bias = torch.randn(n, steps, len(vocab) + 8, device=DEV, generator=g)
    bias[:, :, 3] += 3.0   # "damn" would win everywhere
    for k in range(steps):
        L = P + k
        scores = bias[:, k, :].clone()
        v.mask_completing_tokens_(scores, ids[:, :L].reshape(-1), torch.arange(n + 1, device=DEV) * L)
        ids[:, L] = scores[:, :len(vocab)].argmax(dim=1)
    host = ids.cpu().tolist()
    for row in host:
        prompt = b"".join(vocab[t] for t in row[:P])
        text = prompt + b"".join(vocab[t] for t in row[P:])
        assert all(e <= len(prompt) for _, _, e in ac.find_matches_as_indexes(text, overlapping=True))


def test_two_threads_and_two_automata():
    rng = np.random.default_rng(8)
    v1 = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    pats2 = [b"hello", b"amn", b"c"]
    v2 = BytesAhoCorasick(pats2, matchkind=MatchKind.LeftmostLongest).vocabulary(VOCAB)
    b1, b2 = BruteModel(PATS, VOCAB), BruteModel(pats2, VOCAB)
    hists = _histories(rng, len(VOCAB), 50)
    tokens, offs = _flat(hists)
    errors = []

    def work(v, brute):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(10):
                    logits = torch.zeros(len(hists), len(VOCAB), device=DEV)
                    v.mask_completing_tokens_(logits, tokens, offs)
                    torch.cuda.current_stream().synchronize()
                    got = [torch.isinf(r).nonzero().flatten().tolist() for r in logits]
                    assert got == [brute(h) for h in hists]
        except Exception as e:   # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=work, args=a) for a in ((v1, b1), (v1, b1), (v2, b2))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
