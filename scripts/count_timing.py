"""count_matches_device against scan_device plus diff(match_offsets), per call, on the bench workloads
(device-resident input).

For each workload both answers are computed once and compared: the counts must equal diff(match_offsets) of
scan_device, and, on a sub-sample of the haystacks (a 1 MiB prefix of a single haystack), the CPU oracle's counts.
Then each is timed with CUDA events around back-to-back calls over a window of at least --window-ms, as an exact
answer per call: scan_device (sync=True: it checks that its list is complete) followed by diff(match_offsets), against
count_matches_device.  Prints the card's name and power limit, one JSON line per workload and a table.

    python scripts/count_timing.py [--only c2,c3,c5,c4ll,c4ov,c4full] [--window-ms 400]
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

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402


def scan_counts(ac, d, o, overlapping):
    """The composition count_matches replaces: the whole list, then the difference of its per-haystack offsets."""
    _, mo, _ = ac.scan_device(d, o, overlapping)
    return mo[1:] - mo[:-1]


def oracle_check(ac, pats, kind, overlapping, data, offs, counts, n_sample, seed):
    """counts against the oracle's on a sub-sample of the haystacks; one haystack: the device count of a 1 MiB prefix."""
    nh = len(offs) - 1
    if nh == 1:
        lim = min(int(offs[1]), 1 << 20)
        want = len(Oracle(pats, kind.value).find(data[:lim].tobytes(), overlapping=overlapping))
        d = torch.from_numpy(data[:lim].copy()).cuda()
        return int(ac.count_matches_device(d, torch.tensor([0, lim], device="cuda"), overlapping)[0]) == want
    idx = np.sort(np.random.default_rng(seed).choice(nh, size=min(n_sample, nh), replace=False))
    chunks = [data[offs[i]:offs[i + 1]] for i in idx]
    sub_offs = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=sub_offs[1:])
    _, want, _ = Oracle(pats, kind.value).scan_batch(np.concatenate(chunks), sub_offs, overlapping=overlapping, want_records=False)
    return np.array_equal(want.astype(np.int64), counts[idx])


def workloads(only):
    if "c2" in only:
        pats, data, offs = W.config2()
        yield "config 2 (100 k x 4 KiB), Standard", [p.encode() for p in pats], MatchKind.Standard, False, data, offs
    if "c3" in only:
        pats, data, offs = W.config3()
        yield "config 3 (1 M x 256 B), LeftmostLongest", pats, MatchKind.LeftmostLongest, False, data, offs
    if "c5" in only:
        pats, data, offs = W.config5(n_haystacks=262_144)
        yield "config 5 (256 k x 4 KiB = 1 GiB), Standard", pats, MatchKind.Standard, False, data, offs
    if "c4ll" in only or "c4ov" in only:
        pats, data = W.config4(hay_bytes=1 << 30)
        one = np.array([0, len(data)], dtype=np.int64)
        if "c4ll" in only:
            yield "config 4 (one 1 GiB haystack), LeftmostLongest", pats, MatchKind.LeftmostLongest, False, data, one
        if "c4ov" in only:
            yield "config 4 (one 1 GiB haystack), overlapping", pats, MatchKind.Standard, True, data, one
    if "c4full" in only:
        pats, data = W.config4()
        yield "config 4 (one 4 GiB haystack), overlapping, windows", pats, MatchKind.Standard, True, data, np.array([0, len(data)], dtype=np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c2,c3,c5,c4ll,c4ov,c4full")
    ap.add_argument("--window-ms", type=float, default=400.0)
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    only = set(args.only.split(","))
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows_out = []
    for name, pats, kind, overlapping, data, offs in workloads(only):
        t0 = time.time()
        ac = BytesAhoCorasick(pats, kind)
        d, o = torch.from_numpy(data).cuda(), torch.from_numpy(offs).cuda()
        ref = scan_counts(ac, d, o, overlapping).cpu().numpy()
        scan_engine = ac._ac.last_stats["engine"]
        got = ac.count_matches_device(d, o, overlapping).cpu().numpy()
        st = dict(ac._ac.last_stats)
        ok_ref = bool(np.array_equal(got, ref))
        ok_orc = bool(oracle_check(ac, pats, kind, overlapping, data, offs, got, args.sample, seed=1))
        t_scan, n_scan = per_call_ms(lambda: scan_counts(ac, d, o, overlapping), args.window_ms)
        t_count, n_count = per_call_ms(lambda: ac.count_matches_device(d, o, overlapping), args.window_ms)
        row = {"workload": name, "bytes": int(data.nbytes), "haystacks": int(len(offs) - 1), "matches": int(got.sum()),
               "scan_engine": scan_engine, "count_stats": st, "scan_diff_ms": round(t_scan, 4), "count_matches_device_ms": round(t_count, 4),
               "calls": [n_scan, n_count], "speedup": round(t_scan / t_count, 3), "counts_eq_scan": ok_ref, "counts_eq_oracle_sample": ok_orc,
               "card": info, "setup_s": round(time.time() - t0, 1)}
        rows_out.append(row)
        print(json.dumps(row), flush=True)
        del d, o, ac
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit_w']} W; ms per call (an exact answer each), device-resident input")
    print(f"{'workload':56s} {'engine':>7s} {'scan+diff':>10s} {'count':>10s} {'x':>8s} {'long':>5s}  checks")
    for r in rows_out:
        print(f"{r['workload']:56s} {r['count_stats'].get('engine') or '?':>7s} {r['scan_diff_ms']:10.3f} {r['count_matches_device_ms']:10.3f} "
              f"{r['speedup']:8.2f} {r['count_stats'].get('long_stretches', 0):5d}  {'ok' if r['counts_eq_scan'] and r['counts_eq_oracle_sample'] else 'FAILED'}")
    if not all(r["counts_eq_scan"] and r["counts_eq_oracle_sample"] for r in rows_out):
        sys.exit(1)


if __name__ == "__main__":
    main()
