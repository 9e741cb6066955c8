"""Match masks: match_mask_device against what a user builds without it -- scan_device's rows, then a difference array
(index_add_ of +1 at every start and -1 at every end, cumsum, > 0).  Workloads:

  config4      one 256 MiB haystack of config 4, overlapping (the sieve's cover mode)
  config3      64 MiB of config 3 log lines, LeftmostLongest (the list scan and the mask epilogue)
  config5      16 384 x 4 KiB haystacks of config 5, both searches
  config2      config 2 text (the table walker's rows, OR-ed with acb_mask_rows)
  tokens       4 096 x 2 048 token ids against 256 sequences of 1-4 ids, overlapping
  sets         4 096 haystacks of config 3 text (16 KiB lines, 64 MiB), each with its own random 1 % of the patterns, LeftmostLongest

Every answer is compared with the baseline's before it is timed.  Times are CUDA events around back-to-back calls over a
window of at least --window-ms.  Prints the card's name and power limit, then one JSON line per measurement.

    python scripts/match_mask_timing.py [--window-ms 300] [--only config4,config3,...]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind, TokenAhoCorasick  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402


def emit(name, **kw):
    print(json.dumps({"measure": name, **kw}), flush=True)


def diff_array(scan, n_bytes, offsets):
    """The baseline: rows of scan() (haystack-relative byte positions), +1 / -1 at the ends, cumsum, > 0."""
    m, _, _ = scan()
    m = m.long()
    base = offsets[m[:, 0]]
    acc = torch.zeros(n_bytes + 1, dtype=torch.int32, device=offsets.device)
    ones = torch.ones(m.shape[0], dtype=torch.int32, device=offsets.device)
    acc.index_add_(0, base + m[:, 2], ones)
    acc.index_add_(0, base + m[:, 3], -ones)
    return torch.cumsum(acc[:-1], 0) > 0


def compare(name, ac, mask_fn, base_fn, args, **kw):
    got = mask_fn()
    stats = dict(ac._ac.last_stats)
    want = base_fn()
    same = bool(torch.equal(got, want))
    a, _ = per_call_ms(base_fn, args.window_ms)
    b, _ = per_call_ms(mask_fn, args.window_ms)
    emit(name, **kw, engine=stats.get("engine"), long_stretches=stats.get("long_stretches"), list_records=stats.get("list_records"),
         covered=int(got.sum().item()), baseline_ms=round(a, 3), match_mask_ms=round(b, 3), speedup=round(a / b, 2), same=same)
    if not same:
        raise SystemExit(f"{name}: the mask differs from the baseline")


def bytes_workload(name, ac, data, offs, overlapping, args, **kw):
    dev = torch.device("cuda", 0)
    d = torch.from_numpy(data).to(dev)
    o = torch.from_numpy(offs).to(dev) if offs is not None else torch.tensor([0, data.size], dtype=torch.int64, device=dev)
    compare(name, ac, lambda: ac.match_mask_device(d, o, overlapping),
            lambda: diff_array(lambda: ac._ac.scan_device(d, o, overlapping, False), d.numel(), o), args,
            bytes=int(data.size), haystacks=int(o.numel() - 1), overlapping=overlapping, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--only", default="config4,config3,config5,config2,tokens,sets")
    args = ap.parse_args()
    only = args.only.split(",")
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    if "config4" in only:
        pats, data = W.config4(hay_bytes=256 << 20)
        bytes_workload("config4", BytesAhoCorasick(pats), data, None, True, args, kind="Standard")
    if "config3" in only:
        pats, data, offs = W.config3(n_lines=262_144)
        bytes_workload("config3", BytesAhoCorasick(pats, matchkind=MatchKind.LeftmostLongest), data, offs, False, args,
                       kind="LeftmostLongest")
    if "config5" in only:
        pats, data, offs = W.config5(n_haystacks=16_384)
        ac = BytesAhoCorasick(pats)
        for overlapping in (True, False):
            bytes_workload("config5", ac, data, offs, overlapping, args, kind="Standard")
    if "config2" in only:
        pats, data, offs = W.config2(100_000)
        bytes_workload("config2", AhoCorasick(pats), data, offs, False, args, kind="Standard")
    if "tokens" in only:
        rng = np.random.default_rng(2)
        seqs = [rng.integers(0, 500, size=int(rng.integers(1, 5))).tolist() for _ in range(256)]
        tac = TokenAhoCorasick(seqs)
        n, L = 4096, 2048
        toks = torch.from_numpy(rng.integers(0, 500, size=n * L)).to(dev)
        o = torch.arange(n + 1, dtype=torch.int64, device=dev) * L

        def base():
            m, _, _ = tac.scan_device(toks, o, True)
            m = m.long()
            acc = torch.zeros(toks.numel() + 1, dtype=torch.int32, device=dev)
            ones = torch.ones(m.shape[0], dtype=torch.int32, device=dev)
            acc.index_add_(0, o[m[:, 0]] + m[:, 2], ones)
            acc.index_add_(0, o[m[:, 0]] + m[:, 3], -ones)
            return torch.cumsum(acc[:-1], 0) > 0
        compare("tokens", tac, lambda: tac.match_mask_device(toks, o, True), base, args, tokens=n * L, haystacks=n, sequences=len(seqs),
                overlapping=True, kind="Standard")
    if "sets" in only:
        pats, data, offs = W.config3(n_lines=4096, line_bytes=16384)
        ac = BytesAhoCorasick(pats, matchkind=MatchKind.LeftmostLongest)
        rng = np.random.default_rng(5)
        masks = torch.from_numpy(rng.random((4096, len(pats))) < 0.01).to(dev)
        ps = ac.pattern_sets(masks, device=dev)
        si = torch.arange(4096, dtype=torch.int32, device=dev)
        d, o = torch.from_numpy(data).to(dev), torch.from_numpy(offs).to(dev)
        compare("sets", ac, lambda: ac.match_mask_device(d, o, False, pattern_sets=ps, set_index=si),
                lambda: diff_array(lambda: ac._ac.scan_device(d, o, False, False, flt=(ps, si)), d.numel(), o), args,
                bytes=int(data.size), haystacks=4096, kind="LeftmostLongest", set_fraction=0.01)


if __name__ == "__main__":
    main()
