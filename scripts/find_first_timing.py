"""find_first_device against scan_device plus each haystack's first row, per call, on the bench workloads
(device-resident input).

For each workload both answers are computed once and compared: find_first_device's rows must equal the first row of
every haystack's scan_device list, and, on a sub-sample of the haystacks (a 1 MiB prefix of a single haystack), the
CPU oracle's first records.  Then each is timed with CUDA events around back-to-back calls over a window of at least
--window-ms, as an exact answer per call: scan_device (sync=True: it checks that its list is complete) followed by the
gather of row match_offsets[h], against find_first_device.  Prints the card's name and power limit, one JSON line per
workload and a table.

    python scripts/find_first_timing.py [--only c2,c3,c5,c4] [--window-ms 400]
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


def scan_first_rows(ac, d, o):
    """The composition find_first replaces: the whole list, then row match_offsets[h] where the count is positive."""
    m, mo, total = ac.scan_device(d, o)
    n = o.numel() - 1
    rows = torch.full((n, 3), -1, dtype=torch.int64, device=d.device)
    if total:
        first = m[mo[:-1].clamp(max=total - 1), 1:4].to(torch.int64)
        rows = torch.where((mo[1:] > mo[:-1])[:, None], first, rows)
    return rows


def oracle_check(pats, kind, data, offs, rows, n_sample, seed):
    """rows against the oracle's first records on a sub-sample of the haystacks (a 1 MiB prefix of a single haystack)."""
    nh = len(offs) - 1
    if nh == 1:
        lim = min(int(offs[1]), 1 << 20)
        first = Oracle(pats, kind.value).find(data[:lim].tobytes())
        # a first match that ends inside the prefix is the haystack's first match for every kind but LeftmostLongest,
        # where a longer one may run past the prefix: then only its start is known to be right
        if not first:
            return rows[0][0] < 0 or rows[0][2] > lim - max(len(p) for p in pats)
        want = list(first[0])
        return rows[0].tolist() == want or (kind == MatchKind.LeftmostLongest and rows[0][1] == want[1])
    idx = np.sort(np.random.default_rng(seed).choice(nh, size=min(n_sample, nh), replace=False))
    chunks = [data[offs[i]:offs[i + 1]] for i in idx]
    sub_offs = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=sub_offs[1:])
    _, counts, rec = Oracle(pats, kind.value).scan_batch(np.concatenate(chunks), sub_offs)
    want = np.full((len(idx), 3), -1, dtype=np.int64)
    at = np.concatenate([[0], np.cumsum(counts.astype(np.int64))[:-1]])
    has = counts > 0
    want[has] = rec[at[has]][:, 1:4].astype(np.int64)
    return np.array_equal(want, rows[idx])


def workloads(only):
    if "c2" in only:
        pats, data, offs = W.config2()
        yield "config 2 (100 k x 4 KiB), Standard", [p.encode() for p in pats], MatchKind.Standard, data, offs
    if "c3" in only:
        pats, data, offs = W.config3()
        yield "config 3 (1 M x 256 B), LeftmostLongest", pats, MatchKind.LeftmostLongest, data, offs
    if "c5" in only:
        pats, data, offs = W.config5(n_haystacks=262_144)
        yield "config 5 (256 k x 4 KiB = 1 GiB), Standard", pats, MatchKind.Standard, data, offs
    if "c4" in only:
        pats, data = W.config4(hay_bytes=1 << 30)
        yield "config 4 (one 1 GiB haystack), LeftmostLongest", pats, MatchKind.LeftmostLongest, data, np.array([0, len(data)], dtype=np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c2,c3,c5,c4")
    ap.add_argument("--window-ms", type=float, default=400.0)
    ap.add_argument("--sample", type=int, default=2000)
    args = ap.parse_args()
    only = set(args.only.split(","))
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows_out = []
    for name, pats, kind, data, offs in workloads(only):
        t0 = time.time()
        ac = BytesAhoCorasick(pats, kind)
        d, o = torch.from_numpy(data).cuda(), torch.from_numpy(offs).cuda()
        ref = scan_first_rows(ac, d, o).cpu().numpy()
        scan_engine = ac._ac.last_stats["engine"]
        got = ac.find_first_device(d, o).cpu().numpy()
        st = {k: (v.tolist() if torch.is_tensor(v) else v) for k, v in ac._ac.last_stats.items()}
        ok_ref = bool(np.array_equal(got, ref))
        ok_orc = bool(oracle_check(pats, kind, data, offs, got, args.sample, seed=1))
        t_scan, n_scan = per_call_ms(lambda: scan_first_rows(ac, d, o), args.window_ms)
        t_first, n_first = per_call_ms(lambda: ac.find_first_device(d, o), args.window_ms)
        row = {"workload": name, "bytes": int(data.nbytes), "haystacks": int(len(offs) - 1),
               "with_match": int((got[:, 0] >= 0).sum()), "scan_engine": scan_engine, "first_stats": st,
               "scan_first_rows_ms": round(t_scan, 4), "find_first_device_ms": round(t_first, 4), "calls": [n_scan, n_first],
               "speedup": round(t_scan / t_first, 3), "rows_eq_scan": ok_ref, "rows_eq_oracle_sample": ok_orc,
               "card": info, "setup_s": round(time.time() - t0, 1)}
        rows_out.append(row)
        print(json.dumps(row), flush=True)
        del d, o, ac
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit_w']} W; ms per call (an exact answer each), device-resident input")
    print(f"{'workload':50s} {'engine':>7s} {'scan+rows':>10s} {'find_first':>11s} {'x':>9s} {'matched':>9s}  checks")
    for r in rows_out:
        print(f"{r['workload']:50s} {r['first_stats'].get('engine', '?'):>7s} {r['scan_first_rows_ms']:10.3f} {r['find_first_device_ms']:11.3f} "
              f"{r['speedup']:9.2f} {r['with_match']:9d}  {'ok' if r['rows_eq_scan'] and r['rows_eq_oracle_sample'] else 'FAILED'}")
    if not all(r["rows_eq_scan"] and r["rows_eq_oracle_sample"] for r in rows_out):
        sys.exit(1)


if __name__ == "__main__":
    main()
