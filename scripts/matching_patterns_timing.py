"""matching_patterns_device against scan_device plus torch.unique over haystack * n_patterns + pattern, per call, on
the bench workloads (device-resident input).

For each workload both answers are computed once and compared with each other, and the hits of a sub-sample of the
haystacks (a 1 MiB prefix of a single haystack) with Counter of the CPU oracle's records.  Then each is timed with CUDA
events around back-to-back calls over a window of at least --window-ms, as an exact answer per call: scan_device
(sync=True: it checks that its list is complete) followed by unique, against matching_patterns_device.  Prints the
card's name and power limit, one JSON line per workload and a table.

    python scripts/matching_patterns_timing.py [--only c2,c3,c5,c4ll,c4ov,hot] [--window-ms 400]
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

from ahocorasick_rs_b200 import BytesAhoCorasick, _capi  # noqa: E402
from oracle import Oracle  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402
from scripts.pattern_counts_timing import workloads  # noqa: E402


def scan_unique(ac, d, o, overlapping):
    """The composition matching_patterns replaces: the whole list, then the distinct (haystack, pattern) keys."""
    m, _, _ = ac.scan_device(d, o, overlapping)
    P = ac._ac.n_patterns
    keys, counts = torch.unique(m[:, 0].long() * P + m[:, 1].long(), return_counts=True)
    row_offsets = torch.searchsorted(keys, torch.arange(o.numel(), dtype=torch.int64, device=d.device) * P)
    return row_offsets, keys % P, counts


def oracle_check(ac, pats, kind, overlapping, data, offs, n_sample, seed):
    """The device's hits of a sub-sample of the haystacks (one haystack: a 1 MiB prefix) against the oracle's."""
    nh = len(offs) - 1
    if nh == 1:
        chunks = [data[:min(int(offs[1]), 1 << 20)]]
    else:
        idx = np.sort(np.random.default_rng(seed).choice(nh, size=min(n_sample, nh), replace=False))
        chunks = [data[offs[i]:offs[i + 1]] for i in idx]
    sub_offs = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=sub_offs[1:])
    sub = np.concatenate(chunks)
    _, _, rec = Oracle(pats, kind.value).scan_batch(sub, sub_offs, overlapping=overlapping)
    keys, counts = np.unique(rec[:, 0].astype(np.int64) * len(pats) + rec[:, 1].astype(np.int64), return_counts=True)
    ro, p, c = ac.matching_patterns_device(torch.from_numpy(sub).cuda(), torch.from_numpy(sub_offs).cuda(), overlapping)
    return (np.array_equal(p.cpu().numpy(), keys % len(pats)) and np.array_equal(c.cpu().numpy(), counts) and
            np.array_equal(ro.cpu().numpy(), np.searchsorted(keys, np.arange(len(sub_offs)) * len(pats))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c2,c3,c5,c4ll,c4ov,hot")
    ap.add_argument("--window-ms", type=float, default=400.0)
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    only = set(args.only.split(","))
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows_out = []
    for name, pats, kind, overlapping, data, offs in workloads(only):
        _capi.set_tuning(5 if name.endswith(", sieve") else 0)
        t0 = time.time()
        ac = BytesAhoCorasick(pats, kind)
        d, o = torch.from_numpy(data).cuda(), torch.from_numpy(offs).cuda()
        ref = [t.cpu().numpy() for t in scan_unique(ac, d, o, overlapping)]
        scan_engine = ac._ac.last_stats["engine"]
        got = [t.cpu().numpy() for t in ac.matching_patterns_device(d, o, overlapping)]
        st = dict(ac._ac.last_stats)
        ok_ref = all(np.array_equal(a, b) for a, b in zip(got, ref))
        ok_orc = bool(oracle_check(ac, pats, kind, overlapping, data, offs, args.sample, seed=1))
        t_scan, n_scan = per_call_ms(lambda: scan_unique(ac, d, o, overlapping), args.window_ms)
        t_mp, n_mp = per_call_ms(lambda: ac.matching_patterns_device(d, o, overlapping), args.window_ms)
        row = {"workload": name, "bytes": int(data.nbytes), "haystacks": int(len(offs) - 1), "patterns": len(pats),
               "hits": int(len(got[1])), "matches": int(got[2].sum()), "scan_engine": scan_engine, "stats": st,
               "scan_unique_ms": round(t_scan, 4), "matching_patterns_ms": round(t_mp, 4), "calls": [n_scan, n_mp],
               "speedup": round(t_scan / t_mp, 3), "eq_scan": ok_ref, "eq_oracle_sample": ok_orc, "card": info,
               "setup_s": round(time.time() - t0, 1)}
        rows_out.append(row)
        print(json.dumps(row), flush=True)
        del d, o, ac
        torch.cuda.empty_cache()
    _capi.set_tuning(0)
    print(f"\n{info['name']}, power limit {info['power_limit_w']} W; ms per call (an exact answer each), device-resident input")
    print(f"{'workload':66s} {'engine':>7s} {'scan+unique':>12s} {'matching':>9s} {'x':>8s} {'rows':>5s}  checks")
    for r in rows_out:
        print(f"{r['workload']:66s} {r['stats'].get('engine') or '?':>7s} {r['scan_unique_ms']:12.3f} {r['matching_patterns_ms']:9.3f} "
              f"{r['speedup']:8.2f} {r['stats'].get('rows', 0):5d}  {'ok' if r['eq_scan'] and r['eq_oracle_sample'] else 'FAILED'}")
    if not all(r["eq_scan"] and r["eq_oracle_sample"] for r in rows_out):
        sys.exit(1)


if __name__ == "__main__":
    main()
