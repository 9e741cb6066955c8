"""is_match_device against scan_device, per call, on the bench workloads (device-resident input).

For each workload both calls are warmed up, then each is timed with CUDA events around back-to-back calls over a
window of at least --window-ms, twice: enqueued only (sync=False), and as an exact answer per call (sync=True;
scan_device then checks that its list is complete, and the caller compares its match offsets).  Every mask is checked against diff(match_offsets) > 0 of scan_device, and a
sub-sample of the haystacks against the CPU oracle's counts.  Prints the card's name and power limit, one JSON line per
workload and a table.

    python scripts/is_match_timing.py [--only c2,c3,c5,c4,c3-other] [--window-ms 400]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402


def card():
    try:
        row = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def per_call_ms(fn, window_ms):
    """Mean time of one call: back-to-back calls between two events, repeated until the window is covered."""
    fn()
    fn()
    torch.cuda.synchronize()
    n, total = 1, 0.0
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        total = e0.elapsed_time(e1)
        if total >= window_ms:
            return total / n, n
        n = max(2 * n, int(n * window_ms / max(total, 1e-3)) + 1)


def oracle_check(pats, kind, data, offs, mask, n_sample, seed):
    """The mask against the oracle's counts on a sub-sample of the haystacks (a 1 MiB prefix of a single haystack)."""
    nh = len(offs) - 1
    if nh == 1:
        lim = min(int(offs[1]), 1 << 20)
        _, counts, _ = Oracle(pats, kind.name).scan_batch(data[:lim], np.array([0, lim], dtype=np.int64), want_records=False)
        return bool(counts[0] > 0) <= bool(mask[0])   # a match in the prefix implies True
    idx = np.sort(np.random.default_rng(seed).choice(nh, size=min(n_sample, nh), replace=False))
    chunks = [data[offs[i]:offs[i + 1]] for i in idx]
    sub_offs = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=sub_offs[1:])
    _, counts, _ = Oracle(pats, kind.name).scan_batch(np.concatenate(chunks), sub_offs, want_records=False)
    return np.array_equal(counts > 0, mask[idx])


def workloads(only):
    if "c2" in only:
        pats, data, offs = W.config2()
        yield "config 2 (100 k x 4 KiB)", [p.encode() for p in pats], MatchKind.Standard, data, offs
    c3 = None
    if "c3" in only or "c3-other" in only:
        c3 = W.config3()
    if "c3" in only:
        yield "config 3 (1 M x 256 B)", c3[0], MatchKind.Standard, c3[1], c3[2]
    if "c5" in only:
        pats, data, offs = W.config5(n_haystacks=262_144)
        yield "config 5 (256 k x 4 KiB = 1 GiB)", pats, MatchKind.Standard, data, offs
    if "c4" in only:
        pats, data = W.config4(hay_bytes=1 << 30)
        yield "config 4 (one 1 GiB haystack, LeftmostLongest)", pats, MatchKind.LeftmostLongest, data, np.array([0, len(data)], dtype=np.int64)
    if "c3-other" in only:
        other = W.config3(n_patterns=10_000, n_lines=1, seed=1003)[0]
        yield "config 3 lines, patterns of another seed", other, MatchKind.Standard, c3[1], c3[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c2,c3,c5,c4,c3-other")
    ap.add_argument("--window-ms", type=float, default=400.0)
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    only = set(args.only.split(","))
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = []
    for name, pats, kind, data, offs in workloads(only):
        t0 = time.time()
        ac = BytesAhoCorasick(pats, kind)
        d, o = torch.from_numpy(data).cuda(), torch.from_numpy(offs).cuda()
        _, mo, total = ac.scan_device(d, o)
        ref = (mo[1:] > mo[:-1]).cpu().numpy()
        scan_engine = ac._ac.last_stats["engine"]
        mask = ac.is_match_device(d, o).cpu().numpy()
        st = dict(ac._ac.last_stats)
        ok_ref = bool(np.array_equal(mask, ref))
        ok_orc = bool(oracle_check(pats, kind, data, offs, mask, args.sample, seed=1))
        # enqueue only (sync=False; the workspace already has room for the whole list, and is_match_device's
        # table-walker path waits for its scan whatever sync says)
        t_scan, n_scan = per_call_ms(lambda: ac.scan_device(d, o, sync=False), args.window_ms)
        t_any, n_any = per_call_ms(lambda: ac.is_match_device(d, o, sync=False), args.window_ms)
        # an exact answer per call: scan_device(sync=True) checks that its list is complete, then the comparison
        t_scan_s, _ = per_call_ms(lambda: (lambda r: r[1][1:] > r[1][:-1])(ac.scan_device(d, o)), args.window_ms)
        t_any_s, _ = per_call_ms(lambda: ac.is_match_device(d, o), args.window_ms)
        row = {"workload": name, "bytes": int(data.nbytes), "haystacks": int(len(offs) - 1), "matches": int(total),
               "true": int(mask.sum()), "scan_engine": scan_engine, "any_stats": st,
               "scan_device_ms": round(t_scan, 4), "is_match_device_ms": round(t_any, 4), "calls": [n_scan, n_any],
               "speedup": round(t_scan / t_any, 3), "sync_scan_device_ms": round(t_scan_s, 4),
               "sync_is_match_device_ms": round(t_any_s, 4), "sync_speedup": round(t_scan_s / t_any_s, 3), "mask_eq_scan": ok_ref, "mask_eq_oracle_sample": ok_orc,
               "card": info, "setup_s": round(time.time() - t0, 1)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del d, o, ac
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit_w']} W; ms per call, device-resident input")
    print("sync=False: enqueued back to back; sync=True: an exact answer per call (scan_device + diff > 0)")
    print(f"{'workload':48s} {'engine':>7s} {'scan':>9s} {'is_match':>9s} {'x':>8s} {'scan/sync':>10s} {'is_m/sync':>10s} {'x':>8s} {'true':>9s}  checks")
    for r in rows:
        print(f"{r['workload']:48s} {r['any_stats'].get('engine', '?'):>7s} {r['scan_device_ms']:9.3f} {r['is_match_device_ms']:9.3f} "
              f"{r['speedup']:8.2f} {r['sync_scan_device_ms']:10.3f} {r['sync_is_match_device_ms']:10.3f} {r['sync_speedup']:8.2f} "
              f"{r['true']:9d}  {'ok' if r['mask_eq_scan'] and r['mask_eq_oracle_sample'] else 'FAILED'}")
    if not all(r["mask_eq_scan"] and r["mask_eq_oracle_sample"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
