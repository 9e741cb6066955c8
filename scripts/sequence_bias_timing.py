"""Per-pattern biases for completing tokens: bias_completing_tokens_ against a vectorised torch baseline of the
sequence-bias logits processor, and against mask_completing_tokens_ on the same inputs.

Workload (that of scripts/completions_timing.py): n rows (64, 256) of random histories (128 or 32 768 ids; half of the
rows end in some sequence's p[:-1]), a Llama-3-sized vocabulary (V = 128 256) of bfloat16 logits, 100 or 10 000
sequences of 1-6 ids, and 1 or 16 pattern sets (each set holds a random half of the sequences; rows pick a set at
random).  The biases are multiples of 1/4 in [-8, 8], so every partial sum is exact in float32 and the baseline's
order of accumulation cannot change its result: the outputs are compared bit for bit, and the script stops on any
difference.

Baseline: for every length l, compare the last l - 1 ids of every row with every sequence of that length, AND with the
row's set, accumulate the matching sequences' biases into a float32 (n, V) tensor with index_put_(accumulate=True),
then (logits.float() + bias).to(bfloat16) -- no host round trip.  Times are CUDA events around back-to-back calls over
a window of at least --window-ms.  Prints the card's name and power limit, then one JSON line per measurement.

    python scripts/sequence_bias_timing.py [--window-ms 300]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import TokenAhoCorasick  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402

V = 128256


def emit(measure, **kw):
    print(json.dumps({"measure": measure, **kw}), flush=True)


class Baseline:
    """The patterns grouped by length: (l, P_l x l ids, their global ids)."""

    def __init__(self, pats, dev):
        self.groups = []
        by_len = {}
        for pid, p in enumerate(pats):
            by_len.setdefault(len(p), []).append(pid)
        for l, pids in sorted(by_len.items()):
            self.groups.append((l, torch.tensor([pats[i] for i in pids], dtype=torch.int64, device=dev),
                                torch.tensor(pids, dtype=torch.int64, device=dev)))

    def __call__(self, logits, ids2d, admit, bias):
        """logits (n, V) bfloat16, ids2d (n, H) histories of equal length, admit (n, P) bool, bias (P,) float32."""
        n = logits.shape[0]
        acc = torch.zeros(n, logits.shape[1], dtype=torch.float32, device=logits.device)
        for l, seqs, pids in self.groups:
            hit = admit[:, pids]
            if l > 1:
                hit = hit & (ids2d[:, ids2d.shape[1] - (l - 1):, None] == seqs[:, :l - 1].T[None]).all(dim=1)
            rows, k = hit.nonzero(as_tuple=True)
            acc.index_put_((rows, seqs[k, l - 1]), bias[pids[k]], accumulate=True)
        return (logits.float() + acc).to(logits.dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    emit("card", **card())
    for n_pats in (100, 10000):
        rng = np.random.default_rng(n_pats)
        pats = [[int(x) for x in rng.integers(0, V, int(rng.integers(1, 7)))] for _ in range(n_pats)]
        tac = TokenAhoCorasick(pats)
        base = Baseline(pats, dev)
        bias = torch.tensor(rng.integers(-32, 33, n_pats) / 4.0, dtype=torch.float32, device=dev)
        for n_sets in (1, 16):
            sets = [[p for p in range(n_pats) if rng.random() < 0.5] for _ in range(n_sets)] if n_sets > 1 else [list(range(n_pats))]
            ps = tac.pattern_sets(sets)
            member = torch.zeros(n_sets, n_pats, dtype=torch.bool, device=dev)
            for g, s in enumerate(sets):
                member[g, torch.tensor(s, dtype=torch.int64, device=dev)] = True
            for n in (64, 256):
                set_index = torch.tensor(rng.integers(0, n_sets, n), dtype=torch.int32, device=dev)
                admit = member[set_index.long()]
                for hist_len in (128, 32768):
                    ids = rng.integers(0, V, (n, hist_len))
                    for i in range(0, n, 2):
                        p = pats[int(rng.integers(0, n_pats))]
                        if len(p) > 1:
                            ids[i, hist_len - len(p) + 1:] = p[:-1]
                    ids2d = torch.tensor(ids, dtype=torch.int64, device=dev)
                    flat = ids2d.reshape(-1)
                    offsets = torch.arange(n + 1, device=dev) * hist_len
                    logits0 = torch.randn(n, V, device=dev).to(torch.bfloat16)
                    got = tac.bias_completing_tokens_(logits0.clone(), flat, offsets, bias, pattern_sets=ps, set_index=set_index)
                    want = base(logits0, ids2d, admit, bias)
                    same = bool(torch.equal(got.view(torch.int16), want.view(torch.int16)))
                    biased = int((got.view(torch.int16) != logits0.view(torch.int16)).sum().item())
                    work = logits0.clone()
                    t_base, _ = per_call_ms(lambda: base(work, ids2d, admit, bias), args.window_ms)
                    t_ours, _ = per_call_ms(lambda: tac.bias_completing_tokens_(work, flat, offsets, bias, pattern_sets=ps,
                                                                                set_index=set_index), args.window_ms)
                    t_mask, _ = per_call_ms(lambda: tac.mask_completing_tokens_(work, flat, offsets, pattern_sets=ps, set_index=set_index),
                                            args.window_ms)
                    extra = {}
                    if n_sets == 1:   # the same answer without a filter
                        plain = tac.bias_completing_tokens_(logits0.clone(), flat, offsets, bias)
                        same = same and bool(torch.equal(plain.view(torch.int16), want.view(torch.int16)))
                        t_plain, _ = per_call_ms(lambda: tac.bias_completing_tokens_(work, flat, offsets, bias), args.window_ms)
                        extra = {"unfiltered_ms": round(t_plain, 4)}
                    emit("bias_completing_tokens_", rows=n, vocab=V, dtype="bfloat16", patterns=n_pats, sets=n_sets,
                         history=hist_len, changed_per_row=round(biased / n, 1), baseline_ms=round(t_base, 4),
                         kernel_ms=round(t_ours, 4), mask_ms=round(t_mask, 4), speedup=round(t_base / t_ours, 1),
                         over_mask=round(t_ours / t_mask, 2), **extra, same=same)
                    if not same:
                        raise SystemExit("bias_completing_tokens_ differs from the baseline")


if __name__ == "__main__":
    main()
