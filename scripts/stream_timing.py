"""Times the stream search (StreamBatch.feed_device) against scan_device on the same bytes held whole, on one GPU.
Prints one JSON line per workload: ms per feed, GB/s of the feeds, and scan_device's ms and GB/s over the whole data.
Every number is read with the card's name and power limit, printed first.

  python scripts/stream_timing.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ahocorasick_rs_b200 import AhoCorasick, BytesAhoCorasick, MatchKind  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402


def timed(fn, reps):
    fn()   # warm-up: images, workspaces, module loads
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def streams(ac, d, n, per, step, overlapping, reps):
    """n streams of `per` bytes laid out one after another in d, fed `step` bytes per stream per feed."""
    feeds = -(-per // step)
    # each feed's chunks side by side in one buffer, gathered before the clock starts (one stream: views of d)
    args = []
    for f in range(feeds):
        a, b = f * step, min(per, (f + 1) * step)
        chunk = d[: n * per].view(n, per)[:, a:b].reshape(-1) if n > 1 else d[a:b]
        args.append((chunk, torch.arange(n + 1, dtype=torch.int64, device="cuda") * (b - a),
                     torch.full((n,), f == feeds - 1, dtype=torch.bool, device="cuda")))

    def run():
        sb = ac.stream_batch(n, overlapping)
        for chunk, o, last in args:
            sb.feed_device(chunk, o, last)

    return timed(run, reps), feeds


def whole(ac, d, n, per, overlapping, reps):
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda") * per
    return timed(lambda: ac.scan_device(d[: n * per], offs, overlapping), reps)


def report(name, n, per, step, t_stream, feeds, t_whole):
    total = n * per
    print(json.dumps({"workload": name, "streams": n, "bytes": total, "step_bytes_per_stream": step, "feeds": feeds,
                      "stream_ms_per_feed": round(1e3 * t_stream / feeds, 3), "stream_GBps": round(total / t_stream / 1e9, 1),
                      "scan_device_ms": round(1e3 * t_whole, 3), "scan_device_GBps": round(total / t_whole / 1e9, 1),
                      "stream_over_scan_device": round(t_stream / t_whole, 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)

    pats3, data3, _ = W.config3(n_lines=1 << 21)   # 512 MiB: 512 KiB per stream, three feeds each
    d3 = torch.from_numpy(data3).cuda()
    ac3 = BytesAhoCorasick(pats3, MatchKind.LeftmostLongest)
    n, per = 1024, len(data3) // 1024
    t, feeds = streams(ac3, d3, n, per, 200_000, False, args.reps)
    report("config3 LeftmostLongest, 1024 streams", n, per, 200_000, t, feeds, whole(ac3, d3, n, per, False, args.reps))
    n, per = 4096, len(data3) // 4096
    t, feeds = streams(ac3, d3, n, per, 16 << 10, False, args.reps)
    report("config3 LeftmostLongest, 4096 streams x 16 KiB", n, per, 16 << 10, t, feeds, whole(ac3, d3, n, per, False, args.reps))
    del d3

    pats4 = W.random_lowercase_patterns(100_000, 5, 8, 4)
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    d4 = torch.randint(97, 123, (1 << 30,), dtype=torch.uint8, device="cuda", generator=g)
    ac4 = BytesAhoCorasick(pats4)
    t_whole = whole(ac4, d4, 1, 1 << 30, True, args.reps)
    for step in (64 << 20, 256 << 20):
        t, feeds = streams(ac4, d4, 1, 1 << 30, step, True, args.reps)
        report("config4 overlapping, one stream", 1, 1 << 30, step, t, feeds, t_whole)
    ac4l = BytesAhoCorasick(pats4, MatchKind.LeftmostLongest)
    t, feeds = streams(ac4l, d4, 1, 1 << 30, 64 << 20, False, 1)
    report("config4 LeftmostLongest, one stream", 1, 1 << 30, 64 << 20, t, feeds, whole(ac4l, d4, 1, 1 << 30, False, 1))
    # the str class: code points are counted by one warp per stream, up to its last released row
    acs = AhoCorasick([p.decode() for p in pats4])
    t, feeds = streams(acs, d4, 1, 256 << 20, 64 << 20, True, 1)
    report("config4 overlapping, one AhoCorasick stream (code points)", 1, 256 << 20, 64 << 20, t, feeds,
           whole(acs, d4, 1, 256 << 20, True, 1))


if __name__ == "__main__":
    main()
