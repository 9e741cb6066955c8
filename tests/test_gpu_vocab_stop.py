"""Vocabulary stop strings on the GPU: TokenVocabulary.find_stop_device against the brute force over the oracle (every
id width, scalar and tensor `new`, offset and break edges, AhoCorasick with non-ASCII patterns, every match kind, pattern
sets), the new = 1 identity with mask_completing_tokens_ and the torch-decode plus scan_device path at the 10 000-pattern,
128 256-entry workload, out= in place, CUDA-graph replay, a generation loop checked on the decoded text, and two threads."""
import threading

import numpy as np
import pytest
import torch

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, workloads as W

from .vocab_stop_model import BruteStop

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
PATS = [b"damn", b"\nUser:", b"ab", b"bca", b"aaaa", b"\xc3\xa9t\xc3\xa9", b"ca", b"bca"]
VOCAB = [b"d", b"am", b"n", b"damn", b"\n", b"User", b":", b"hello", b"", b"a", b"b", b"c", b"ab", b"xxbcaxx", b"\xc3", b"\xa9t",
         b"\xc3\xa9", b"t", b"aa", b""]


def _flat(hists, dtype=torch.int64):
    offs = np.zeros(len(hists) + 1, dtype=np.int64)
    np.cumsum([len(h) for h in hists], out=offs[1:])
    npt = {torch.uint16: np.uint16, torch.int32: np.int32, torch.int64: np.int64}[dtype]
    flat = np.concatenate([np.asarray(h, dtype=np.int64) for h in hists] + [np.zeros(0, dtype=np.int64)]).astype(npt)
    return torch.from_numpy(flat).to(DEV), torch.from_numpy(offs).to(DEV)


def _histories(rng, n_vocab, n, breaks=(-1, -7, None, None, 1 << 20)):
    out = [[], [-1], [n_vocab], [0, 1, 2], [4, 5, 6], [4, -1, 5, 6], [14, 15, 14, 16, 17, 14, 16], [9, 9, 9, 9], [12, 11, 9],
           [19, 8, 0, 8, 1, 8, 2], [13], [10, 11, 9, 8, 8]]
    for i in range(n):
        h = [int(x) for x in rng.integers(0, n_vocab, int(rng.integers(0, 14)))]
        if i % 3 == 0 and h:
            b = rng.choice([x for x in breaks if x is not None] + [n_vocab, n_vocab + 100])
            h.insert(int(rng.integers(0, len(h) + 1)), int(b))
        out.append(h)
    return out


def _rows(res):
    return [None if r[0] < 0 else tuple(r) for r in res.cpu().tolist()]


@pytest.mark.parametrize("tdtype", [torch.uint16, torch.int32, torch.int64])
def test_against_the_model_every_width_scalar_and_tensor_new(tdtype):
    rng = np.random.default_rng(1)
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    hists = _histories(rng, len(VOCAB), 60, breaks=(None,) if tdtype == torch.uint16 else (-1, -7, 1 << 20))
    tokens, offs = _flat(hists, tdtype)
    for k in (0, 1, 2, 5, 100):
        got = _rows(v.find_stop_device(tokens, offs, new=k))
        assert got == [brute(h, k) for h in hists], k
        assert v.last_stats["mode"] == "vocab_stop" and v.last_stats["n_vocab"] == len(VOCAB)
    news = [int(x) for x in rng.integers(-3, 8, len(hists))]
    got = _rows(v.find_stop_device(tokens, offs, new=torch.tensor(news, device=DEV)))
    assert got == [brute(h, k) for h, k in zip(hists, news)]


def test_offset_edges_and_long_histories():
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    rng = np.random.default_rng(2)
    flat = [int(x) for x in rng.integers(-2, len(VOCAB) + 2, 100_000)]
    flat[-3:] = [0, 1, 2]
    tokens = torch.tensor(flat, dtype=torch.int64, device=DEV)
    n = len(flat)
    offsets = [5, 2, 40, 40, -9, 7, n + 50, 99_990, n, 0, n]   # clamped, decreasing, offsets[0] > 0
    got = _rows(v.find_stop_device(tokens, torch.tensor(offsets, device=DEV), new=3))

    def clamp(o):
        return min(max(o, 0), n)

    want = []
    for i in range(len(offsets) - 1):
        a, b = clamp(offsets[i]), clamp(offsets[i + 1])
        want.append(brute(flat[a:b] if b >= a else [], 3))
    assert got == want
    assert got[-1] == (0, n - 1, 1, 4)   # the 100 000-id history ends in "damn"


def test_ac_non_ascii_and_every_match_kind():
    pats = ["é", "naïve", "日本語", "na"]
    vocab = [b"na", b"\xc3", b"\xaf", b"ve", b"\xa9", "日".encode(), "本語".encode()[:2], "本語".encode()[2:], b""]
    enc = [p.encode() for p in pats]
    brute = BruteStop(enc, vocab)
    hists = [[1, 4], [0, 1, 2, 3], [5, 6, 8, 7], [0, 1, 8, 2, 3], [5, -1, 6, 7], [1, 8, 8, 4]]
    tokens, offs = _flat(hists)
    outs = []
    for kind in MatchKind:
        v = AhoCorasick(pats, matchkind=kind).vocabulary(vocab)
        for k in (1, 2):
            got = _rows(v.find_stop_device(tokens, offs, new=k))
            assert got == [brute(h, k) for h in hists], (kind, k)
            outs.append(got)
    assert outs[0][0] == (0, 1, 1, 2) and outs[0][1] == (1, 3, 2, 6) and outs[0][2] == (2, 3, 4, 9)
    v = AhoCorasick(pats, matchkind=MatchKind.LeftmostFirst).vocabulary(vocab)
    assert v.find_stop([0, 1, 2, 3], new=1) == (1, 3, 2, 6)


def test_pattern_sets_with_far_out_of_range_indices():
    rng = np.random.default_rng(3)
    ac = BytesAhoCorasick(PATS)
    v = ac.vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    sets = [[0, 1], [2, 3, 7], [], list(range(len(PATS))), [6], [3]]
    ps = ac.pattern_sets(sets)
    hists = _histories(rng, len(VOCAB), 40)
    tokens, offs = _flat(hists)
    idx = [int(x) for x in rng.integers(0, len(sets), len(hists))]
    for i, bad in zip(range(0, len(hists), 7), (-1, len(sets), (1 << 31), (1 << 62), (1 << 63) - 1, -(1 << 63))):
        idx[i] = bad
    got = _rows(v.find_stop_device(tokens, offs, new=2, pattern_sets=ps, set_index=torch.tensor(idx, device=DEV)))
    want = [brute(h, 2, set(sets[s])) if 0 <= s < len(sets) else None for h, s in zip(hists, idx)]
    assert got == want
    # the host forms: patterns= per history, token indexes mapped back to the caller's history
    want = [brute(h, 2, set(sets[i % len(sets)])) for i, h in enumerate(hists)]
    assert v.find_stop_batch(hists, 2, [sets[i % len(sets)] for i in range(len(hists))]) == want


def test_out_in_place_and_host_forms():
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    hists = [[7] * 50 + [0, 1, 2], [4, 5, 6], [], [9, 9, 9, 9, 9]]
    tokens, offs = _flat(hists)
    out = torch.full((4, 4), 99, dtype=torch.int64, device=DEV)
    r = v.find_stop_device(tokens, offs, 1, out=out)
    assert r.data_ptr() == out.data_ptr() and _rows(out) == [brute(h, 1) for h in hists]
    assert v.find_stop([7] * 50 + [0, 1, 2]) == (0, 52, 1, 4)
    assert v.find_stop_batch(hists, [1, 3, 1, 2]) == [brute(h, k) for h, k in zip(hists, [1, 3, 1, 2])]
    with pytest.raises(TypeError, match="out"):
        v.find_stop_device(tokens, offs, 1, out=torch.zeros(4, 4, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="rows"):
        v.find_stop_device(tokens, offs, 1, out=torch.zeros(3, 4, dtype=torch.int64, device=DEV))
    with pytest.raises(TypeError, match="new"):
        v.find_stop_device(tokens, offs, torch.ones(4, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="new"):
        v.find_stop_device(tokens, offs, torch.ones(3, dtype=torch.int64, device=DEV))
    with pytest.raises(ValueError, match="new"):
        v.find_stop_device(tokens, offs, -1)
    # per-history counts: beyond int64 is the whole history; a CUDA tensor belongs to the device form
    assert v.find_stop_batch([[0, 1, 2], [4, 5, 6]], [1 << 70, 0]) == [brute([0, 1, 2], 3), None]
    with pytest.raises(TypeError, match="find_stop_device"):
        v.find_stop_batch(hists, torch.ones(4, dtype=torch.int64, device=DEV))
    # no patterns, no vocabulary: all -1 / None
    assert BytesAhoCorasick([b"zz"]).vocabulary([]).find_stop_batch([[0, 1], []]) == [None, None]
    e = BytesAhoCorasick([b"zz"]).vocabulary([])
    assert _rows(e.find_stop_device(tokens, offs, 2)) == [None] * 4


def test_one_launch_per_call_and_none_for_no_rows():
    from ahocorasick_rs_b200 import _capi
    L = _capi.lib()
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    tokens, offs = _flat([[0, 1, 2], [4, 5, 6]])
    v.find_stop_device(tokens, offs, 1)   # the first call uploads the image
    out = torch.empty((2, 4), dtype=torch.int64, device=DEV)
    news = torch.ones(2, dtype=torch.int64, device=DEV)
    for new in (1, news):
        before = L.acb_launch_count()
        v.find_stop_device(tokens, offs, new, out=out)
        assert L.acb_launch_count() == before + 1
    before = L.acb_launch_count()
    empty = v.find_stop_device(tokens, offs[:1], 1)
    assert L.acb_launch_count() == before and empty.shape == (0, 4)
    torch.cuda.synchronize()
    assert _rows(out) == [(0, 2, 1, 4), (1, 2, 1, 6)]


def _scale_case():
    names = W.patterns_long()
    pats = names + [" " + n for n in names] + [n + " " for n in names]
    pats = [p.encode() for p in pats[:10000]]
    rng = np.random.default_rng(11)
    text = (W.haystack_template() + " ".join(names[int(i)] for i in rng.integers(0, len(names), 20000))).encode()
    vocab = [bytes([b]) for b in range(256)]
    for k, a in zip(rng.integers(2, 9, 128256 - 256), rng.integers(0, len(text) - 8, 128256 - 256)):
        vocab.append(text[int(a):int(a) + int(k)])
    return pats, vocab, text, rng


def _tokenize(text, a, n_bytes, index):
    h, p = [], a
    while p < a + n_bytes:   # a greedy tokenization of a slice of the text
        k = next(k for k in range(8, 0, -1) if text[p:p + k] in index)
        h.append(index[text[p:p + k]])
        p += k
    return h


@pytest.mark.parametrize("n_sets", [1, 16])
def test_scale_identity_with_the_mask(n_sets):
    """new = 1: row h + [t] has a stop exactly when mask_completing_tokens_ bans t after h, for every candidate t."""
    pats, vocab, text, rng = _scale_case()
    ac = BytesAhoCorasick(pats)
    v = ac.vocabulary(vocab)
    index = {s: t for t, s in enumerate(vocab)}
    hists = [_tokenize(text, int(rng.integers(0, len(text) - 200)), int(rng.integers(0, 100)), index) for _ in range(6)]
    sets = [[p for p in range(len(pats)) if rng.random() < 0.5] for _ in range(n_sets)]
    ps = ac.pattern_sets(sets) if n_sets > 1 else None
    idx = torch.tensor(rng.integers(0, n_sets, len(hists)), device=DEV) if n_sets > 1 else None
    logits = torch.zeros(len(hists), len(vocab), device=DEV)
    tokens, offs = _flat(hists, torch.int32)
    v.mask_completing_tokens_(logits, tokens, offs, ps, idx)
    V = len(vocab)
    cand = torch.arange(V, dtype=torch.int32, device=DEV)
    for i, h in enumerate(hists):
        hist = torch.tensor(h, dtype=torch.int32, device=DEV)
        rows = torch.cat([hist.repeat(V, 1), cand[:, None]], 1).reshape(-1)   # V rows: h + [t]
        roffs = torch.arange(V + 1, dtype=torch.int64, device=DEV) * (len(h) + 1)
        kw = {} if n_sets == 1 else dict(pattern_sets=ps, set_index=idx[i].repeat(V))
        res = v.find_stop_device(rows, roffs, 1, **kw)
        assert torch.equal(res[:, 0] >= 0, torch.isinf(logits[i])), i
        assert bool((res[res[:, 0] >= 0][:, 1] == len(h)).all())


def test_scale_against_torch_decode_and_scan():
    pats, vocab, text, rng = _scale_case()
    ac = BytesAhoCorasick(pats)
    v = ac.vocabulary(vocab)
    index = {s: t for t, s in enumerate(vocab)}
    need = ac._ac.max_pattern_len - 1
    hists = [_tokenize(text, int(rng.integers(0, len(text) - 300)), int(rng.integers(1, 200)), index) for _ in range(48)]
    news = [int(x) for x in rng.integers(1, 17, len(hists))]
    tokens, offs = _flat(hists, torch.int32)
    got = _rows(v.find_stop_device(tokens, offs, torch.tensor(news, device=DEV)))
    # the second path: each row's bytes decoded with torch ops, one scan_device(overlapping=True), the stop picked on the host
    lens = torch.tensor([len(x) for x in vocab], device=DEV)
    starts = torch.cumsum(lens, 0) - lens
    blob = torch.from_numpy(np.frombuffer(b"".join(vocab), dtype=np.uint8).copy()).to(DEV)
    ids = tokens.long()
    ln = lens[ids]
    seg = torch.repeat_interleave(torch.arange(ids.numel(), device=DEV), ln)
    first = torch.cumsum(ln, 0) - ln
    data = blob[starts[ids][seg] + torch.arange(seg.numel(), device=DEV) - first[seg]]
    row_bytes = torch.tensor([sum(len(vocab[t]) for t in h) for h in hists], device=DEV)
    hoffs = torch.zeros(len(hists) + 1, dtype=torch.int64, device=DEV)
    hoffs[1:] = torch.cumsum(row_bytes, 0)
    m, _, _ = ac.scan_device(data, hoffs, overlapping=True)
    m = m.cpu().numpy()
    for i, (h, k) in enumerate(zip(hists, news)):
        ends = np.cumsum([len(vocab[t]) for t in h])
        k = min(k, len(h))
        new_from = int(ends[len(h) - k - 1]) if len(h) > k else 0
        best = None
        for _, p, s, e in m[m[:, 0] == i]:
            if e > new_from:
                key = (e, -(e - s), p)
                best = key if best is None or key < best else best
        if best is None:
            assert got[i] is None, i
            continue
        e, p = int(best[0]), int(best[2])
        tok = int(np.searchsorted(ends, e - 1, side="right"))
        assert got[i] == (p, tok, e - int(ends[tok] - len(vocab[h[tok]])), len(pats[p])), i
    assert any(g is not None for g in got) and need > 0


def test_cuda_graph_replay():
    ac = BytesAhoCorasick(PATS)
    v = ac.vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    sets = ac.pattern_sets([[0, 1, 2], [3, 4, 5, 6, 7], list(range(len(PATS)))])
    rng = np.random.default_rng(9)
    L = 8
    tokens = torch.zeros(16 * L, dtype=torch.int64, device=DEV)
    offs = torch.arange(17, dtype=torch.int64, device=DEV) * L
    news = torch.ones(16, dtype=torch.int64, device=DEV)
    idx = torch.zeros(16, dtype=torch.int64, device=DEV)
    out = torch.empty((16, 4), dtype=torch.int64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        v.find_stop_device(tokens, offs, news, sets, idx, out=out)   # warm-up: uploads the image
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        v.find_stop_device(tokens, offs, news, sets, idx, out=out)
    all_sets = [{0, 1, 2}, {3, 4, 5, 6, 7}, set(range(len(PATS)))]
    for _ in range(4):
        h = rng.integers(-1, len(VOCAB), (16, L))
        k = rng.integers(-1, 6, 16)
        si = rng.integers(-1, 4, 16)
        tokens.copy_(torch.from_numpy(h.reshape(-1)))
        news.copy_(torch.from_numpy(k))
        idx.copy_(torch.from_numpy(si))
        g.replay()
        torch.cuda.synchronize()
        want = [brute(h[i].tolist(), int(k[i]), all_sets[si[i]]) if 0 <= si[i] < 3 else None for i in range(16)]
        assert _rows(out) == want


def test_generation_loop_with_per_row_stop_sets():
    """64 rows x 64 argmax steps over random logits; each row has its own stop set.  The first step that reports a stop
    agrees with the overlapping search of the row's decoded text."""
    pats = [b"ab", b"\nUser:", b"cab", b"bb", b"User", b"a:"]
    vocab = [b"a", b"b", b"c", b"\n", b"Us", b"er", b":", b"ab", b"", b"x", b"er:"]
    ac = BytesAhoCorasick(pats)
    v = ac.vocabulary(vocab)
    sets = [[0, 2], [1], [3, 4], [5], [1, 3]]
    ps = ac.pattern_sets(sets)
    n, steps = 64, 64
    g = torch.Generator(device=DEV).manual_seed(5)
    idx = torch.arange(n, device=DEV) % len(sets)
    prompt = torch.full((n, 1), 9, dtype=torch.int64, device=DEV)
    ids = prompt
    first = [None] * n
    for step in range(steps):
        logits = torch.randn(n, len(vocab), generator=g, device=DEV)
        nxt = logits.argmax(1, keepdim=True)
        ids = torch.cat([ids, nxt], 1)
        res = v.find_stop_device(ids.reshape(-1), torch.arange(n + 1, device=DEV) * ids.shape[1], 1, ps, idx).cpu().tolist()
        for i in range(n):
            if first[i] is None and res[i][0] >= 0:
                first[i] = (step, tuple(res[i]))
    rows = ids.cpu().tolist()
    seen = 0
    for i in range(n):
        text = b"".join(vocab[t] for t in rows[i])
        ends = np.cumsum([len(vocab[t]) for t in rows[i]])
        m = ac.find_matches_as_indexes(text, overlapping=True, patterns=sets[i % len(sets)])
        if not m:
            assert first[i] is None
            continue
        p, s, e = min(m, key=lambda x: (x[2], -(x[2] - x[1]), x[0]))
        tok = int(np.searchsorted(ends, e - 1, side="right"))
        assert first[i] is not None, i
        step, (gp, gt, ge, gl) = first[i]
        assert (step + 1, gp, gt, ge, gl) == (tok, p, tok, e - int(ends[tok] - len(vocab[rows[i][tok]])), e - s), i
        seen += 1
    assert seen > 10


def test_two_threads():
    v = BytesAhoCorasick(PATS).vocabulary(VOCAB)
    brute = BruteStop(PATS, VOCAB)
    errors = []

    def work(seed):
        try:
            rng = np.random.default_rng(seed)
            for _ in range(20):
                hists = _histories(rng, len(VOCAB), 30)
                tokens, offs = _flat(hists)
                k = int(rng.integers(1, 4))
                got = _rows(v.find_stop_device(tokens, offs, k))
                assert got == [brute(h, k) for h in hists]
        except Exception as e:   # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=work, args=(s,)) for s in (1, 2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
