"""Vocabulary masks: TokenVocabulary.mask_completing_tokens_ against the batched overlapping scan a user would otherwise
write.

Workload: n rows (64, 256) of random histories (128 or 32 768 ids of the vocabulary; every other row ends in the first
bytes of some pattern, spelled with one-byte ids), V = 128 256 bfloat16 logits, 100 or 10 000 string patterns of 3-20
bytes (seeded substrings of a text made of the haystack template and the names), and 1 or 16 pattern sets (each set a
random half of the patterns; rows pick a set at random).  The vocabulary: the 256 single bytes, then seeded substrings
of 2-8 bytes of the same text.

Baseline: for each row, the last max_pattern_len - 1 bytes of its text (decoded on the host, outside the timing) are
put in front of every entry, all 128 256 haystacks go through BytesAhoCorasick.scan_device(overlapping=True) in one
batch per 16 rows, and the ids of the matches that end past the row's bytes (and whose pattern the row's set admits)
get -inf.  Its output is compared with the kernel's, bit for bit, before either is timed.  Times are CUDA events around
back-to-back calls over a window of at least --window-ms.  Each kernel's time comes from torch.profiler (CUPTI device
timestamps of 20 further calls): the two kernels run inside one C call, so no event can sit between them.  The share of
(row, id) pairs decided by the first byte (a match, or a state of depth <= 1) is computed from the image on the host.
TokenAhoCorasick.mask_completing_tokens_ (the token-level mask) on the same rows, with 100 or 10 000 id sequences of
1-6 ids, is a point of reference.  Prints the card's name and power limit, then one JSON line per measurement.

    python scripts/vocab_mask_timing.py [--window-ms 300]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import BytesAhoCorasick, TokenAhoCorasick  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402
from tests.vocab_model import MASK, MATCH, VocabImage  # noqa: E402

V = 128256


def emit(measure, **kw):
    print(json.dumps({"measure": measure, **kw}), flush=True)


def corpus(rng):
    names = W.patterns_long()
    return (W.haystack_template() + " ".join(names[int(i)] for i in rng.integers(0, len(names), 20000))).encode()


def substrings(rng, text, n, lo, hi):
    return [text[int(a):int(a) + int(k)] for k, a in zip(rng.integers(lo, hi + 1, n), rng.integers(0, len(text) - hi, n))]


def host_image(v):
    buf = np.zeros(v.image_bytes, dtype=np.uint8)
    rc = v._ac._L.acb_vocab_write(v._ac._h, v._blob.ctypes.data, v._offsets.ctypes.data, v.n_vocab, buf.ctypes.data, v.image_bytes)
    assert rc == 0
    return VocabImage(buf.tobytes())


def first_byte_share(img, states):
    """Share of (row, non-empty id) pairs the first byte decides: a match, or a state of depth <= 1."""
    lens = img.recs[:, 1]
    ne = np.flatnonzero(lens > 0)
    cols = img.colmap[img.bytes[img.recs[ne, 0]]]
    decided = 0
    for s in states:
        e = img.trans[s, cols]
        decided += int(np.count_nonzero((e & MATCH) | ((e & MASK) < img.lvl2)))
    return decided / (len(states) * len(ne))


class Baseline:
    """The batched overlapping scan of T + vocab[t] for every row and id."""

    def __init__(self, ac, vocab, k, dev):
        self.ac, self.k, self.dev = ac, k, dev
        lens = np.array([len(v) for v in vocab], dtype=np.int64)
        self.blob = torch.from_numpy(np.frombuffer(b"".join(vocab), dtype=np.uint8).copy()).to(dev)
        voffs = np.zeros(len(vocab) + 1, dtype=np.int64)
        np.cumsum(lens, out=voffs[1:])
        # one row's batch: haystack t = the row's k bytes, then vocab[t]; index < k reads the row's bytes, k + j blob[j]
        idx = np.empty(len(vocab) * k + int(voffs[-1]), dtype=np.int64)
        hoffs = np.zeros(len(vocab) + 1, dtype=np.int64)
        np.cumsum(lens + k, out=hoffs[1:])
        starts = hoffs[:-1]
        for j in range(k):
            idx[starts + j] = j
        pos = np.arange(int(voffs[-1]), dtype=np.int64)
        owner = np.repeat(np.arange(len(vocab)), lens)
        idx[starts[owner] + k + (pos - voffs[owner])] = k + pos
        self.idx = torch.from_numpy(idx).to(dev)
        self.hoffs = torch.from_numpy(hoffs).to(dev)
        self.per = len(idx)

    def __call__(self, logits, tails, admit, rows_per_batch=16):
        """tails: uint8 (n, k) device tensor of each row's last k bytes; admit: (n, P) bool or None."""
        n, nv = logits.shape[0], self.hoffs.numel() - 1
        for a in range(0, n, rows_per_batch):
            b = min(n, a + rows_per_batch)
            data = torch.cat([tails[a:b], self.blob.expand(b - a, -1)], dim=1).gather(1, self.idx.expand(b - a, -1)).reshape(-1)
            offs = (torch.arange(b - a, device=self.dev)[:, None] * self.per + self.hoffs[None, :-1]).reshape(-1)
            offs = torch.cat([offs, torch.tensor([(b - a) * self.per], device=self.dev)])
            m, _, _ = self.ac.scan_device(data, offs, overlapping=True)
            m = m.to(torch.int64)
            m = m[m[:, 3] > self.k]
            row, tok = a + m[:, 0] // nv, m[:, 0] % nv
            if admit is not None:
                keep = admit[row, m[:, 1]]
                row, tok = row[keep], tok[keep]
            logits[row, tok] = float("-inf")
        return logits


def kernel_times(fn, reps=20):
    """Mean device time per call of each CUDA kernel fn launches (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "vocab_" in ev.key:
            name = "state_kernel_us" if "vocab_state_kernel" in ev.key else "mask_kernel_us"
            total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[name] = round(total / reps, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    emit("card", **card())
    rng = np.random.default_rng(2026)
    text = corpus(rng)
    vocab = [bytes([b]) for b in range(256)] + substrings(rng, text, V - 256, 2, 8)
    for n_pats in (100, 10000):
        prng = np.random.default_rng(n_pats)
        pats = substrings(prng, text, n_pats, 3, 20)
        ac = BytesAhoCorasick(pats)
        v = ac.vocabulary(vocab)
        img = host_image(v)
        k = img.need
        base = Baseline(ac, vocab, k, dev)
        tpats = [[int(x) for x in prng.integers(0, V, int(prng.integers(1, 7)))] for _ in range(n_pats)]
        tac = TokenAhoCorasick(tpats)
        for n_sets in (1, 16):
            sets = [[p for p in range(n_pats) if prng.random() < 0.5] for _ in range(n_sets)] if n_sets > 1 else [list(range(n_pats))]
            ps, tps = ac.pattern_sets(sets), tac.pattern_sets(sets)
            member = torch.zeros(n_sets, n_pats, dtype=torch.bool, device=dev)
            for g, s in enumerate(sets):
                member[g, torch.tensor(s, dtype=torch.int64, device=dev)] = True
            for n in (64, 256):
                set_index = torch.tensor(prng.integers(0, n_sets, n), dtype=torch.int32, device=dev)
                admit = member[set_index.long()] if n_sets > 1 else None
                for hist_len in (128, 32768):
                    ids = prng.integers(256, V, (n, hist_len))
                    for i in range(0, n, 2):   # the first bytes of a pattern, one byte per id
                        p = pats[int(prng.integers(0, n_pats))][:-1]
                        ids[i, hist_len - len(p):] = list(p)
                    tails = np.zeros((n, k), dtype=np.uint8)
                    states = []
                    for i in range(n):
                        tail = b"".join(vocab[t] for t in ids[i, -k:])[-k:] if k else b""
                        tails[i, :] = np.frombuffer(tail, dtype=np.uint8)
                        states.append(img.state(ids[i, -k:].tolist()))
                    ids2d = torch.tensor(ids, dtype=torch.int64, device=dev)
                    flat = ids2d.reshape(-1)
                    offsets = torch.arange(n + 1, device=dev) * hist_len
                    dtails = torch.from_numpy(tails).to(dev)
                    logits0 = torch.randn(n, V, device=dev).to(torch.bfloat16)
                    kw = dict(pattern_sets=ps, set_index=set_index) if n_sets > 1 else {}
                    got = v.mask_completing_tokens_(logits0.clone(), flat, offsets, **kw)
                    want = base(logits0.clone(), dtails, admit)
                    same = bool(torch.equal(got.view(torch.int16), want.view(torch.int16)))
                    banned = int(torch.isinf(got).sum().item())
                    if not same:   # name the first differing pairs, with the oracle's and the image interpreter's answers
                        from oracle import Oracle
                        orc = Oracle(pats, "Standard")
                        diff = torch.nonzero(got.view(torch.int16) != want.view(torch.int16)).tolist()
                        for r, t in diff[:8]:
                            ok = (lambda p: True) if admit is None else (lambda p, r=r: bool(admit[r, p]))
                            T = tails[r].tobytes()
                            truth = any(e > k and ok(p) for p, _, e in orc.find(T + vocab[t], overlapping=True))
                            adm = None if admit is None else set(torch.nonzero(admit[r]).flatten().tolist())
                            emit("mismatch", row=r, id=t, kernel=bool(torch.isinf(got[r, t])), baseline=bool(torch.isinf(want[r, t])),
                                 oracle=truth, interpreter=img.banned(states[r], t, adm), tail=T.hex(), entry=vocab[t].hex(),
                                 set=int(set_index[r]))
                        emit("mismatch", patterns=n_pats, sets=n_sets, rows=n, history=hist_len, differing=len(diff))
                        raise SystemExit("mask_completing_tokens_ differs from the baseline")
                    work = logits0.clone()
                    call = lambda: v.mask_completing_tokens_(work, flat, offsets, **kw)  # noqa: E731
                    t_ours, _ = per_call_ms(call, args.window_ms)
                    t_base, _ = per_call_ms(lambda: base(work, dtails, admit), args.window_ms)
                    tkw = dict(pattern_sets=tps, set_index=set_index) if n_sets > 1 else {}
                    t_tok, _ = per_call_ms(lambda: tac.mask_completing_tokens_(work, flat, offsets, **tkw), args.window_ms)
                    emit("vocab_mask_completing_tokens_", rows=n, vocab=V, dtype="bfloat16", patterns=n_pats, sets=n_sets,
                         history=hist_len, banned_per_row=round(banned / n, 1), baseline_ms=round(t_base, 4),
                         kernel_ms=round(t_ours, 4), speedup=round(t_base / t_ours, 1), **kernel_times(call),
                         first_byte_share=round(first_byte_share(img, states), 4), tail_hit_ids=int(v.last_stats["tail_hit_ids"]),
                         token_mask_ms=round(t_tok, 4), same=same)


if __name__ == "__main__":
    main()
