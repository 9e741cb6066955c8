"""count_matches_by_pattern_device against scan_device plus torch.bincount of its pattern column, per call, on the
bench workloads (device-resident input).

For each workload both answers are computed once and compared with each other, and the per-pattern counts of a
sub-sample of the haystacks (a 1 MiB prefix of a single haystack) with the CPU oracle's histogram.  Then each is timed
with CUDA events around back-to-back calls over a window of at least --window-ms, as an exact answer per call:
scan_device (sync=True: it checks that its list is complete) followed by bincount, against
count_matches_by_pattern_device.  Prints the card's name and power limit, one JSON line per workload and a table.

    python scripts/pattern_counts_timing.py [--only c2,c3,c5,c4ll,c4ov,hot] [--window-ms 400]
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

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, _capi  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from oracle import Oracle  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402


def scan_bincount(ac, d, o, overlapping):
    """The composition count_matches_by_pattern replaces: the whole list, then a histogram of its pattern column."""
    m, _, _ = ac.scan_device(d, o, overlapping)
    return torch.bincount(m[:, 1].long(), minlength=ac._ac.n_patterns)


def oracle_check(ac, pats, kind, overlapping, data, offs, n_sample, seed):
    """The device's per-pattern counts of a sub-sample of the haystacks (one haystack: a 1 MiB prefix) against the
    oracle's histogram of the same bytes."""
    nh = len(offs) - 1
    if nh == 1:
        lim = min(int(offs[1]), 1 << 20)
        chunks = [data[:lim]]
    else:
        idx = np.sort(np.random.default_rng(seed).choice(nh, size=min(n_sample, nh), replace=False))
        chunks = [data[offs[i]:offs[i + 1]] for i in idx]
    sub_offs = np.zeros(len(chunks) + 1, dtype=np.int64)
    np.cumsum([len(c) for c in chunks], out=sub_offs[1:])
    sub = np.concatenate(chunks)
    _, _, rec = Oracle(pats, kind.value).scan_batch(sub, sub_offs, overlapping=overlapping)
    want = np.bincount(rec[:, 1].astype(np.int64), minlength=len(pats))
    got = ac.count_matches_by_pattern_device(torch.from_numpy(sub).cuda(), torch.from_numpy(sub_offs).cuda(), overlapping)
    return np.array_equal(got.cpu().numpy(), want)


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
    if "hot" in only:
        # one single-byte pattern that matches every position of 64 MiB, and a few rare ones: every lane of every
        # verification round adds to the same counter.  The engine rule would pick the table walker for this text, so
        # the sieve is forced (kernel 5): this workload measures the pattern mode's atomics
        rng = np.random.default_rng(6)
        data = np.full(64 << 20, ord("a"), dtype=np.uint8)
        pos = rng.choice(len(data) - 8, size=1000, replace=False)
        for k, p in enumerate(pos):
            data[p:p + 5] = np.frombuffer([b"xqzjk", b"vwxyz", b"zzqzz"][k % 3], dtype=np.uint8)
        pats = [b"a", b"xqzjk", b"vwxyz", b"zzqzz", b"qqqqq"]
        one = np.array([0, len(data)], dtype=np.int64)
        yield "hot pattern (64 MiB, one byte matches everywhere), overlapping, sieve", pats, MatchKind.Standard, True, data, one


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
        ref = scan_bincount(ac, d, o, overlapping).cpu().numpy()
        scan_engine = ac._ac.last_stats["engine"]
        got = ac.count_matches_by_pattern_device(d, o, overlapping).cpu().numpy()
        st = dict(ac._ac.last_stats)
        ok_ref = bool(np.array_equal(got, ref))
        ok_orc = bool(oracle_check(ac, pats, kind, overlapping, data, offs, args.sample, seed=1))
        t_scan, n_scan = per_call_ms(lambda: scan_bincount(ac, d, o, overlapping), args.window_ms)
        t_pc, n_pc = per_call_ms(lambda: ac.count_matches_by_pattern_device(d, o, overlapping), args.window_ms)
        row = {"workload": name, "bytes": int(data.nbytes), "haystacks": int(len(offs) - 1), "patterns": len(pats),
               "matches": int(got.sum()), "scan_engine": scan_engine, "stats": st, "scan_bincount_ms": round(t_scan, 4),
               "pattern_counts_ms": round(t_pc, 4), "calls": [n_scan, n_pc], "speedup": round(t_scan / t_pc, 3),
               "eq_scan": ok_ref, "eq_oracle_sample": ok_orc, "card": info, "setup_s": round(time.time() - t0, 1)}
        rows_out.append(row)
        print(json.dumps(row), flush=True)
        del d, o, ac
        torch.cuda.empty_cache()
    _capi.set_tuning(0)
    print(f"\n{info['name']}, power limit {info['power_limit_w']} W; ms per call (an exact answer each), device-resident input")
    print(f"{'workload':66s} {'engine':>7s} {'scan+bincount':>14s} {'by_pattern':>11s} {'x':>8s} {'long':>5s}  checks")
    for r in rows_out:
        print(f"{r['workload']:66s} {r['stats'].get('engine') or '?':>7s} {r['scan_bincount_ms']:14.3f} {r['pattern_counts_ms']:11.3f} "
              f"{r['speedup']:8.2f} {r['stats'].get('long_stretches', 0):5d}  {'ok' if r['eq_scan'] and r['eq_oracle_sample'] else 'FAILED'}")
    if not all(r["eq_scan"] and r["eq_oracle_sample"] for r in rows_out):
        sys.exit(1)


if __name__ == "__main__":
    main()
