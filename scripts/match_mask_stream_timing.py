"""Match-mask streams: match_mask_stream_batch against what a user builds without it -- stream_batch's rows, then a
torch scatter of their spans (index_add_ of +1 / -1, cumsum) into a window per stream that carries the flags of the
positions not released yet.  Both release the same positions after every feed (R = max(0, F - (max_pattern_len - 1)),
in tokens for token ids); every feed's flags and flag offsets are compared before the clock runs.  Workloads:

  tokens     4 096 token streams, one id per stream per feed (256 feeds), 256 banned sequences of 2-8 ids, Standard and
             overlapping: the generation case, in ms per feed
  config3    config 3 LeftmostLongest, 4 096 streams x 128 KiB in 16 KiB feeds (the stream search's §10 workload)
  config4    config 4's patterns, one overlapping 1 GiB stream in 64 MiB feeds; also match_mask_device on the whole GiB

Times are the best of --reps runs of every feed of a workload, each ending in a device synchronise (both forms read
their released counts on the host after every feed).  Prints the card's name and power limit, then one JSON line per
measurement.

    python scripts/match_mask_stream_timing.py [--reps 3] [--only tokens,config3,config4]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, TokenAhoCorasick  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from scripts.is_match_timing import card  # noqa: E402


def emit(measure, **kw):
    print(json.dumps({"measure": measure, **kw}), flush=True)


class Composition:
    """stream_batch rows scattered into a carried window.  Positions are in the rows' units (bytes, or tokens for a
    token batch, whose tail is k - 1 tokens); `halo` is the tail in those units."""

    def __init__(self, sb, n, halo):
        self.sb, self.n, self.halo = sb, n, halo
        self.fed = torch.zeros(n, dtype=torch.int64, device="cuda")
        self.held = torch.zeros((n, max(halo, 1)), dtype=torch.bool, device="cuda")

    def feed_device(self, data, offsets, last=None):
        n, halo = self.n, self.halo
        rows, _ = self.sb.feed_device(data, offsets, last)
        lens = offsets[1:] - offsets[:-1]
        lastb = last if last is not None else torch.zeros(n, dtype=torch.bool, device="cuda")
        r_old = (self.fed - halo).clamp(min=0)
        t_old = self.fed - r_old
        f_new = self.fed + lens
        r_new = torch.where(lastb, f_new, (f_new - halo).clamp(min=0))
        reg = t_old + lens                 # the window of stream i: its held positions, then its chunk
        reg_off = torch.cumsum(reg, 0) - reg
        total = int(reg.sum().item())
        ar = torch.arange(halo, device="cuda")
        hm = ar[None, :] < t_old[:, None]
        win = torch.zeros(total, dtype=torch.bool, device="cuda")
        win[(reg_off[:, None] + ar[None, :])[hm]] = self.held[:, :halo][hm]
        acc = torch.zeros(total + 1, dtype=torch.int32, device="cuda")
        if rows.shape[0]:
            s = rows[:, 0]
            base = reg_off[s] - r_old[s]
            ones = torch.ones(rows.shape[0], dtype=torch.int32, device="cuda")
            acc.index_add_(0, base + rows[:, 2], ones)
            acc.index_add_(0, base + rows[:, 3], -ones)
        win |= torch.cumsum(acc[:-1], 0) > 0
        stream_of = torch.repeat_interleave(torch.arange(n, device="cuda"), reg, output_size=total)
        rel = torch.arange(total, device="cuda") - reg_off[stream_of]
        out = rel < (r_new - r_old)[stream_of]
        flags = win[out]
        keep = ~out
        held = torch.zeros_like(self.held)
        held[stream_of[keep], rel[keep] - (r_new - r_old)[stream_of[keep]]] = win[keep]
        self.held = held
        self.fed = torch.where(lastb, torch.zeros_like(f_new), f_new)
        fo = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        fo[1:] = torch.cumsum(r_new - r_old, 0)
        return flags, fo, r_old


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def compare_and_time(name, ac, feeds, n, overlapping, halo_units, reps, whole=None, **kw):
    """feeds: [(data, offsets, last)].  Checks every feed of both forms, then times each over all feeds."""
    ms = ac.match_mask_stream_batch(n, overlapping)
    comp = Composition(ac.stream_batch(n, overlapping), n, halo_units)
    released = 0
    for data, offs, last in feeds:
        f, fo, fs = ms.feed_device(data, offs, last)
        g, go, gs = comp.feed_device(data, offs, last)
        if not (torch.equal(f, g) and torch.equal(fo, go) and torch.equal(fs, gs)):
            raise SystemExit(f"{name}: the mask stream differs from the composition")
        if whole is not None and not torch.equal(f, whole[released:released + f.numel()]):
            raise SystemExit(f"{name}: the mask stream differs from match_mask_device of the whole stream")
        released += f.numel()
    stats = dict(ms.last_stats)

    def run(make):
        b = make()
        for data, offs, last in feeds:
            b.feed_device(data, offs, last)

    t_mask = timed(lambda: run(lambda: ac.match_mask_stream_batch(n, overlapping)), reps)
    t_comp = timed(lambda: run(lambda: Composition(ac.stream_batch(n, overlapping), n, halo_units)), reps)
    emit(name, **kw, streams=n, feeds=len(feeds), released=released, covered_last_feed=int(f.sum().item()),
         sieve_task_bytes=stats.get("task_bytes"), mask_stream_ms_per_feed=round(1e3 * t_mask / len(feeds), 3),
         composition_ms_per_feed=round(1e3 * t_comp / len(feeds), 3), speedup=round(t_comp / t_mask, 2), same=True)
    return t_mask


def tokens(reps):
    rng = np.random.default_rng(11)
    vocab, n, steps = 400, 4096, 256
    banned = [rng.integers(0, vocab, size=int(rng.integers(2, 9))).tolist() for _ in range(256)]
    seqs = rng.integers(0, vocab, size=(n, steps))
    for i in range(n):   # some banned sequences in every stream, some cut by the end
        for _ in range(4):
            b = banned[int(rng.integers(0, 256))]
            at = int(rng.integers(0, steps))
            seqs[i, at:at + len(b)] = b[:steps - at]
    ids = torch.from_numpy(seqs).cuda()
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda")
    feeds = [(ids[:, j].contiguous(), offs, torch.full((n,), j == steps - 1, dtype=torch.bool, device="cuda")) for j in range(steps)]
    k = max(len(b) for b in banned)
    for kind, overlapping, name in ((MatchKind.Standard, False, "Standard"), (MatchKind.Standard, True, "overlapping")):
        ac = TokenAhoCorasick(banned, kind)
        compare_and_time(f"tokens {name}", ac, feeds, n, overlapping, k - 1, reps, ids_per_feed=n)


def config3(reps):
    pats, data, _ = W.config3(n_lines=1 << 21)   # 512 MiB: 4 096 streams x 128 KiB
    d = torch.from_numpy(data).cuda()
    ac = BytesAhoCorasick(pats, MatchKind.LeftmostLongest)
    n, per, step = 4096, 128 << 10, 16 << 10
    feeds = []
    for f in range(per // step):
        chunk = d[: n * per].view(n, per)[:, f * step:(f + 1) * step].reshape(-1)
        feeds.append((chunk, torch.arange(n + 1, dtype=torch.int64, device="cuda") * step,
                      torch.full((n,), f == per // step - 1, dtype=torch.bool, device="cuda")))
    t = compare_and_time("config3 LeftmostLongest", ac, feeds, n, False, ac._ac.max_pattern_len - 1, reps, bytes=n * per)
    emit("config3 LeftmostLongest rate", mask_stream_GBps=round(n * per / t / 1e9, 1))


def config4(reps):
    pats, data = W.config4(hay_bytes=1 << 30)
    d = torch.from_numpy(data).cuda()
    ac = BytesAhoCorasick(pats, MatchKind.Standard)
    step = 64 << 20
    offs0 = torch.tensor([0, d.numel()], dtype=torch.int64, device="cuda")
    whole = ac.match_mask_device(d, offs0, True)
    feeds = [(d[a:a + step], torch.tensor([0, step], dtype=torch.int64, device="cuda"),
              torch.tensor([a + step == d.numel()], dtype=torch.bool, device="cuda")) for a in range(0, d.numel(), step)]
    t = compare_and_time("config4 overlapping, one 1 GiB stream", ac, feeds, 1, True, ac._ac.max_pattern_len - 1, reps, whole=whole,
                         bytes=d.numel())
    t_whole = timed(lambda: ac.match_mask_device(d, offs0, True), reps)
    emit("config4 match_mask_device, the whole GiB", ms=round(1e3 * t_whole, 3), mask_stream_total_ms=round(1e3 * t, 3),
         mask_stream_over_whole=round(t / t_whole, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="tokens,config3,config4")
    args = ap.parse_args()
    emit("device", **card())
    for name in args.only.split(","):
        {"tokens": tokens, "config3": config3, "config4": config4}[name](args.reps)


if __name__ == "__main__":
    main()
