"""Times the stream queries (is_match_stream_batch, find_first_stream_batch, count_matches_stream_batch) against the
composition they replace -- the rows stream (stream_batch) with len / [0] / numel() > 0 of each feed's rows -- on the
DESIGN §10 stream workloads, on one GPU.  Both sides are fed the same chunks and their answers are compared after
every feed before anything is timed.  Prints one JSON line per workload; the card's name and power limit come first.

  python scripts/stream_query_timing.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402


def feeds_of(d, n, per, step):
    """Each feed's chunks side by side in one buffer (views of d for one stream), gathered before the clock starts."""
    out = []
    n_feeds = -(-per // step)
    for f in range(n_feeds):
        a, b = f * step, min(per, (f + 1) * step)
        chunk = d[: n * per].view(n, per)[:, a:b].reshape(-1) if n > 1 else d[a:b]
        out.append((chunk, torch.arange(n + 1, dtype=torch.int64, device="cuda") * (b - a),
                    torch.full((n,), f == n_feeds - 1, dtype=torch.bool, device="cuda")))
    return out


def composition(ac, query, n, overlapping, feeds):
    """The rows stream and the answer from its rows: -> a function that runs every feed and returns the answers."""
    def run():
        sb = ac.stream_batch(n, overlapping)
        seen = torch.zeros(n, dtype=torch.int64, device="cuda")
        first = torch.full((n, 3), -1, dtype=torch.int64, device="cuda")
        answers = []
        for chunk, o, last in feeds:
            rows, ro = sb.feed_device(chunk, o, last)
            k = ro[1:] - ro[:-1]
            if query == "find_first":   # rows[0] of each stream's first feed that released one
                new = (seen == 0) & (k > 0)
                first = torch.where(new[:, None], rows[ro[:-1].clamp(max=max(rows.shape[0] - 1, 0)), 1:4] if rows.shape[0] else first, first)
            seen = seen + k
            answers.append(seen > 0 if query == "is_match" else first.clone() if query == "find_first" else seen.clone())
        return answers
    return run


def queries(ac, query, n, overlapping, feeds):
    def run():
        sb = {"is_match": lambda: ac.is_match_stream_batch(n), "find_first": lambda: ac.find_first_stream_batch(n),
              "count": lambda: ac.count_matches_stream_batch(n, overlapping)}[query]()
        answers = [sb.feed_device(chunk, o, last) for chunk, o, last in feeds]
        run.stats = sb.last_stats
        return answers
    return run


def timed(fn, reps):
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def compare(name, ac, query, n, overlapping, feeds, reps, whole=None):
    comp, new = composition(ac, query, n, overlapping, feeds), queries(ac, query, n, overlapping, feeds)
    a, b = comp(), new()   # (also the warm-up)
    for i, (x, y) in enumerate(zip(a, b)):
        if not torch.equal(x, y):
            raise SystemExit(f"{name}: answers differ after feed {i}")
    t_comp, t_new = timed(comp, reps), timed(new, reps)
    total = sum(int(o[-1].item()) for _, o, _ in feeds)
    line = {"workload": name, "query": query, "streams": n, "bytes": total, "feeds": len(feeds),
            "composition_ms_per_feed": round(1e3 * t_comp / len(feeds), 3), "query_ms_per_feed": round(1e3 * t_new / len(feeds), 3),
            "query_GBps": round(total / t_new / 1e9, 1), "speedup": round(t_comp / t_new, 2),
            "stats": {k: v for k, v in new.stats.items() if k in ("tasks_skipped", "windows_skipped", "flagged", "pending", "held",
                                                                  "long_stretches", "records")}}
    if whole is not None:
        t_whole = timed(whole, reps)
        line.update({"whole_ms": round(1e3 * t_whole, 3), "whole_GBps": round(total / t_whole / 1e9, 1)})
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)

    # config 3 as 4 096 LeftmostLongest streams, 16 KiB per stream per feed: most streams match in their first feed
    pats3, data3, _ = W.config3(n_lines=1 << 21)
    d3 = torch.from_numpy(data3).cuda()
    ac3 = BytesAhoCorasick(pats3, MatchKind.LeftmostLongest)
    n, per = 4096, len(data3) // 4096
    f3 = feeds_of(d3, n, per, 16 << 10)
    for query in ("is_match", "find_first", "count"):
        compare("config3 LeftmostLongest, 4096 streams x 16 KiB", ac3, query, n, False, f3, args.reps)
    del d3, f3

    # config 4: one overlapping stream in 64 MiB feeds (count); one LeftmostLongest stream (count on the grid path)
    pats4 = W.random_lowercase_patterns(100_000, 5, 8, 4)
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    d4 = torch.randint(97, 123, (1 << 30,), dtype=torch.uint8, device="cuda", generator=g)
    f4 = feeds_of(d4, 1, 1 << 30, 64 << 20)
    one = torch.tensor([0, 1 << 30], dtype=torch.int64, device="cuda")
    ac4 = BytesAhoCorasick(pats4)
    compare("config4 overlapping, one stream, 64 MiB feeds", ac4, "count", 1, True, f4, args.reps,
            whole=lambda: ac4.count_matches_device(d4, one, overlapping=True))
    ac4l = BytesAhoCorasick(pats4, MatchKind.LeftmostLongest)
    compare("config4 LeftmostLongest, one stream, 64 MiB feeds", ac4l, "count", 1, False, f4, 1,
            whole=lambda: ac4l.count_matches_device(d4, one))


if __name__ == "__main__":
    main()
