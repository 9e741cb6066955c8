"""Pattern sets: the filter's own cost, and what a filtered call saves against the composition it replaces.

  filter cost   config 3 scan_device / find_first_device, config 4 overlapping count_matches_device and config 5
                scan_device, each unfiltered against one set that holds every pattern (the answers must be equal);
  1 % sets      4 096 haystacks of config 3 text, each with its own random 1 % of the patterns: the filtered
                overlapping scan against an unfiltered scan plus a torch mask of the rows (the answers must be equal);
  token stream  find_first_stream_batch over token ids, 4 096 streams fed 16 tokens each per feed, with and without a
                stop list per stream (eight lists of 4 stop sequences out of 256).

Times are CUDA events around back-to-back calls over a window of at least --window-ms.  Prints the card's name and
power limit, then one JSON line per measurement.

    python scripts/pattern_sets_timing.py [--window-ms 300]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ahocorasick_rs_b200 import BytesAhoCorasick, MatchKind, TokenAhoCorasick  # noqa: E402
from ahocorasick_rs_b200 import workloads as W  # noqa: E402
from scripts.is_match_timing import card, per_call_ms  # noqa: E402


def emit(name, **kw):
    print(json.dumps({"measure": name, **kw}), flush=True)


def filter_cost(args, dev):
    n3 = 262_144
    pats, data, offs = W.config3(n_lines=n3)
    d, o = torch.from_numpy(data).to(dev), torch.from_numpy(offs).to(dev)
    for kind in (MatchKind.Standard, MatchKind.LeftmostLongest):
        ac = BytesAhoCorasick(pats, matchkind=kind)
        ps = ac.pattern_sets([range(len(pats))], device=dev)
        si = torch.zeros(n3, dtype=torch.int32, device=dev)
        m0, mo0, t0 = ac.scan_device(d, o)
        m0, mo0 = m0.clone(), mo0.clone()
        m1, mo1, t1 = ac.scan_device(d, o, pattern_sets=ps, set_index=si)
        same = t0 == t1 and torch.equal(m0, m1) and torch.equal(mo0, mo1)
        same = same and torch.equal(ac.find_first_device(d, o), ac.find_first_device(d, o, pattern_sets=ps, set_index=si))
        for q, f0, f1 in (("scan_device", lambda: ac.scan_device(d, o), lambda: ac.scan_device(d, o, pattern_sets=ps, set_index=si)),
                          ("find_first_device", lambda: ac.find_first_device(d, o),
                           lambda: ac.find_first_device(d, o, pattern_sets=ps, set_index=si))):
            a, _ = per_call_ms(f0, args.window_ms)
            b, _ = per_call_ms(f1, args.window_ms)
            emit("filter_cost", workload="config3", bytes=int(data.size), kind=kind.name, query=q, unfiltered_ms=round(a, 3),
                 all_allowed_ms=round(b, 3), ratio=round(b / a, 3), same=bool(same))
    # dense sets: stage 2 is hot
    pats4, data4 = W.config4(hay_bytes=256 << 20)
    d4, o4 = torch.from_numpy(data4).to(dev), torch.tensor([0, data4.size], dtype=torch.int64, device=dev)
    ac = BytesAhoCorasick(pats4)
    ps = ac.pattern_sets([range(len(pats4))], device=dev)
    si = torch.zeros(1, dtype=torch.int32, device=dev)
    same = torch.equal(ac.count_matches_device(d4, o4, True), ac.count_matches_device(d4, o4, True, pattern_sets=ps, set_index=si))
    a, _ = per_call_ms(lambda: ac.count_matches_device(d4, o4, True), args.window_ms)
    b, _ = per_call_ms(lambda: ac.count_matches_device(d4, o4, True, pattern_sets=ps, set_index=si), args.window_ms)
    emit("filter_cost", workload="config4", bytes=int(data4.size), kind="Standard", query="count_matches_device(overlapping)",
         unfiltered_ms=round(a, 3), all_allowed_ms=round(b, 3), ratio=round(b / a, 3), same=bool(same))
    n5 = 16_384
    pats5, data5, offs5 = W.config5(n_haystacks=n5)
    d5, o5 = torch.from_numpy(data5).to(dev), torch.from_numpy(offs5).to(dev)
    ac = BytesAhoCorasick(pats5)
    ps = ac.pattern_sets([range(len(pats5))], device=dev)
    si = torch.zeros(n5, dtype=torch.int32, device=dev)
    m0, mo0, t0 = ac.scan_device(d5, o5)
    m0 = m0.clone()
    m1, _, t1 = ac.scan_device(d5, o5, pattern_sets=ps, set_index=si)
    same = t0 == t1 and torch.equal(m0, m1)
    a, _ = per_call_ms(lambda: ac.scan_device(d5, o5), args.window_ms)
    b, _ = per_call_ms(lambda: ac.scan_device(d5, o5, pattern_sets=ps, set_index=si), args.window_ms)
    emit("filter_cost", workload="config5", bytes=int(data5.size), kind="Standard", query="scan_device", unfiltered_ms=round(a, 3),
         all_allowed_ms=round(b, 3), ratio=round(b / a, 3), same=bool(same))


def one_percent_sets(args, dev):
    pats, data, offs = W.config3(n_lines=262_144)
    n = 4096
    per = (offs.size - 1) // n   # lines per haystack
    offs_h = offs[::per][: n + 1].copy()
    data = data[: offs_h[-1]]
    d, o = torch.from_numpy(data).to(dev), torch.from_numpy(offs_h).to(dev)
    ac = BytesAhoCorasick(pats)
    rng = np.random.default_rng(1)
    mask = torch.from_numpy(rng.random((n, len(pats))) < 0.01).to(dev)
    ps = ac.pattern_sets(mask, device=dev)
    si = torch.arange(n, dtype=torch.int32, device=dev)

    def composed():
        m, mo, total = ac.scan_device(d, o, True)
        m = m.to(torch.int64)
        keep = mask[m[:, 0], m[:, 1]]
        return m[keep]

    def filtered():
        return ac.scan_device(d, o, True, pattern_sets=ps, set_index=si)

    m1 = filtered()[0].to(torch.int64)   # (a copy: the scan's rows are a view of the workspace the next scan reuses)
    same = torch.equal(composed(), m1)
    a, _ = per_call_ms(composed, args.window_ms)
    b, _ = per_call_ms(filtered, args.window_ms)
    emit("one_percent_sets", haystacks=n, bytes=int(data.size), rows=int(m1.shape[0]), composed_ms=round(a, 3), filtered_ms=round(b, 3),
         speedup=round(a / b, 3), same=bool(same))


def token_stream(args, dev):
    rng = np.random.default_rng(2)
    stops = [list(rng.integers(0, 50_000, size=int(rng.integers(1, 5)))) for _ in range(256)]
    ac = TokenAhoCorasick(stops, matchkind=MatchKind.LeftmostFirst)
    n, step = 4096, 16
    lists = [list(rng.choice(256, size=4, replace=False)) for _ in range(8)]
    ps = ac.pattern_sets(lists, device=dev)
    si = torch.from_numpy(rng.integers(0, 8, size=n).astype(np.int32)).to(dev)
    toks = torch.from_numpy(rng.integers(0, 50_000, size=n * step)).to(dev)
    offs = torch.arange(n + 1, dtype=torch.int64, device=dev) * step
    plain = ac.find_first_stream_batch(n)
    sets = ac.find_first_stream_batch(n, pattern_sets=ps, set_index=si)
    a, k = per_call_ms(lambda: plain.feed_device(toks, offs), args.window_ms)
    b, _ = per_call_ms(lambda: sets.feed_device(toks, offs), args.window_ms)
    emit("token_stream_feed", streams=n, tokens_per_feed=step, stop_sequences=len(stops), plain_ms=round(a, 3), per_stream_sets_ms=round(b, 3),
         ratio=round(b / a, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--only", default="cost,sets,tokens")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    only = args.only.split(",")
    if "cost" in only:
        filter_cost(args, dev)
    if "sets" in only:
        one_percent_sets(args, dev)
    if "tokens" in only:
        token_stream(args, dev)


if __name__ == "__main__":
    main()
