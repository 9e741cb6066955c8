"""Vocabulary stop strings: TokenVocabulary.find_stop_device against the torch decode plus batched overlapping scan a
user would otherwise write.

Workload (DESIGN §4.18's): n rows (64, 256, 1 024) of random histories (128 or 32 768 ids of the vocabulary), the last
`new` (1, 4, 16) of them new; every other row holds a whole pattern, spelled with one-byte ids, whose last byte falls on
a random new id.  100 or 10 000 string patterns of 3-20 bytes (seeded substrings of a text made of the haystack template
and the names), and 1 or 16 pattern sets (each a random half of the patterns; rows pick a set at random).  The
vocabulary: the 256 single bytes, then seeded substrings of 2-8 bytes of the same text (V = 128 256; no entry is empty,
so the last max_pattern_len - 1 ids before the new ones hold every byte that can matter).

Baseline: gather those ids and the new ones, decode them with torch ops (entry offsets and lengths, repeat_interleave
into the entry bytes), run the bytes through BytesAhoCorasick.scan_device(overlapping=True) (its output sizing
synchronises), keep the matches ending in new bytes (and admitted by the row's set), and pick each row's earliest end,
then longest, then lowest pid with one scatter_reduce; map the end back to (token, end) with searchsorted.  Its output
is compared with the kernel's, row for row, before either is timed.  Times are CUDA events around back-to-back calls
over a window of at least --window-ms; the kernel's own time is from torch.profiler (20 further calls).  Prints the
card's name and power limit, then one JSON line per measurement.

    python scripts/vocab_stop_timing.py [--window-ms 150]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import BytesAhoCorasick  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402
from scripts.vocab_mask_timing import V, corpus, substrings  # noqa: E402


def emit(measure, **kw):
    print(json.dumps({"measure": measure, **kw}), flush=True)


class Baseline:
    """The torch decode + scan_device(overlapping=True) stop finder for rows of equal length without breaks or empty ids."""

    def __init__(self, ac, pats, vocab, dev):
        self.ac = ac
        lens = np.array([len(v) for v in vocab], dtype=np.int64)
        offs = np.zeros(len(vocab), dtype=np.int64)
        np.cumsum(lens[:-1], out=offs[1:])
        self.lens = torch.from_numpy(lens).to(dev)
        self.offs = torch.from_numpy(offs).to(dev)
        self.blob = torch.from_numpy(np.frombuffer(b"".join(vocab), dtype=np.uint8).copy()).to(dev)
        self.pat_len = torch.tensor([len(p) for p in pats], dtype=torch.int64, device=dev)
        self.need = max(ac._ac.max_pattern_len - 1, 0)

    def __call__(self, ids2d, new, admit):
        n, L = ids2d.shape
        w = min(L, new + self.need)
        win = ids2d[:, L - w:]                                   # the ids that can matter, then the new ones
        ln = self.lens[win]
        cum = ln.cumsum(1)                                       # per row: the bytes up to and including each id
        row_bytes = cum[:, -1]
        new_from = cum[:, w - new - 1] if w > new else torch.zeros_like(row_bytes)
        starts = self.offs[win].reshape(-1)
        flat_len = ln.reshape(-1)
        seg = torch.repeat_interleave(torch.arange(flat_len.numel(), device=ids2d.device), flat_len)
        first = torch.cumsum(flat_len, 0) - flat_len
        idx = starts[seg] + (torch.arange(seg.numel(), device=ids2d.device) - first[seg])
        data = self.blob[idx]
        hoffs = torch.zeros(n + 1, dtype=torch.int64, device=ids2d.device)
        hoffs[1:] = row_bytes.cumsum(0)
        m, _, _ = self.ac.scan_device(data, hoffs, overlapping=True)
        m = m.to(torch.int64)
        hay, pid, s, e = m[:, 0], m[:, 1], m[:, 2], m[:, 3]   # positions within each haystack
        keep = e > new_from[hay]
        if admit is not None:
            keep &= admit[hay, pid]
        hay, pid, s, e = hay[keep], pid[keep], s[keep], e[keep]
        key = (e << 40) | ((0xffff - (e - s)) << 24) | pid      # earliest end, then longest, then lowest pid
        best = torch.full((n,), torch.iinfo(torch.int64).max, dtype=torch.int64, device=ids2d.device)
        best.scatter_reduce_(0, hay, key, "amin")
        hit = best != torch.iinfo(torch.int64).max
        bp = best & 0xffffff
        be = best >> 40
        tw = torch.searchsorted(cum, (be - 1).clamp(min=0).unsqueeze(1), right=True).squeeze(1).clamp(max=w - 1)
        tok_end = be - (cum.gather(1, tw.unsqueeze(1)).squeeze(1) - ln.gather(1, tw.unsqueeze(1)).squeeze(1))
        out = torch.stack([bp, tw + (L - w), tok_end, self.pat_len[bp.clamp(max=self.pat_len.numel() - 1)]], 1)
        return torch.where(hit.unsqueeze(1), out, torch.full_like(out, -1))


def kernel_us(fn, reps=20):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "vocab_stop_kernel" in ev.key:
            total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            return round(total / reps, 2)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=150.0)
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
        base = Baseline(ac, pats, vocab, dev)
        for n_sets in (1, 16):
            sets = [[p for p in range(n_pats) if prng.random() < 0.5] for _ in range(n_sets)] if n_sets > 1 else [list(range(n_pats))]
            ps = ac.pattern_sets(sets)
            member = torch.zeros(n_sets, n_pats, dtype=torch.bool, device=dev)
            for g, s in enumerate(sets):
                member[g, torch.tensor(s, dtype=torch.int64, device=dev)] = True
            for n in (64, 256, 1024):
                set_index = torch.tensor(prng.integers(0, n_sets, n), dtype=torch.int32, device=dev)
                admit = member[set_index.long()] if n_sets > 1 else None
                kw = dict(pattern_sets=ps, set_index=set_index) if n_sets > 1 else {}
                for hist_len in (128, 32768):
                    for new in (1, 4, 16):
                        ids = prng.integers(256, V, (n, hist_len))
                        for i in range(0, n, 2):   # a whole pattern whose last byte falls on a new id
                            p = pats[int(prng.integers(0, n_pats))]
                            at = hist_len - int(prng.integers(0, new))
                            ids[i, at - len(p):at] = list(p)
                        ids2d = torch.tensor(ids, dtype=torch.int64, device=dev)
                        flat = ids2d.reshape(-1)
                        offsets = torch.arange(n + 1, device=dev) * hist_len
                        out = torch.empty((n, 4), dtype=torch.int64, device=dev)
                        got = v.find_stop_device(flat, offsets, new, out=out, **kw).clone()
                        want = base(ids2d, new, admit)
                        same = bool(torch.equal(got, want))
                        if not same:
                            bad = torch.nonzero((got != want).any(1)).flatten().tolist()
                            for r in bad[:8]:
                                emit("mismatch", row=r, kernel=got[r].tolist(), baseline=want[r].tolist(), set=int(set_index[r]))
                            raise SystemExit(f"find_stop_device differs from the baseline on {len(bad)} rows")
                        call = lambda: v.find_stop_device(flat, offsets, new, out=out, **kw)  # noqa: E731
                        t_ours, _ = per_call_ms(call, args.window_ms)
                        t_base, _ = per_call_ms(lambda: base(ids2d, new, admit), args.window_ms)
                        emit("vocab_find_stop_device", rows=n, vocab=V, patterns=n_pats, sets=n_sets, history=hist_len, new=new,
                             stops=int((got[:, 0] >= 0).sum()), baseline_ms=round(t_base, 4), call_ms=round(t_ours, 4),
                             kernel_us=kernel_us(call), speedup=round(t_base / t_ours, 1), same=same)


if __name__ == "__main__":
    main()
