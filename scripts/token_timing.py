"""Times TokenAhoCorasick on one GPU: seeded Zipf-distributed ids over a 128,256-id vocabulary, generated on the device,
256 k documents x 2,048 int32 tokens (1.5 GiB encoded, one call below WINDOW_BYTES), 100 k 13-gram patterns, half of
them drawn from the data.  Reports the encode kernel alone (CUDA events over many launches: GB/s of algorithmic bytes,
7 per int32 id, and its share of 3.35 TB/s), the whole-step tokens/s of scan_device, count_matches_device and
is_match_device with the share of each step spent encoding, and the per-feed latency of find_first_stream_batch.  A
sample of documents is checked against the oracle in the same run.  Prints one JSON line per measurement; the card's
name and power limit come first.

  python scripts/token_timing.py [--docs 262144] [--tokens 2048] [--patterns 100000] [--reps 5]
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
from ahocorasick_rs_b200 import MatchKind, TokenAhoCorasick, _capi  # noqa: E402
from oracle import Oracle  # noqa: E402

VOCAB = 128_256
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def zipf_ids(n, gen, s=1.1):
    """n ids, rank r drawn with probability ~ r^-s, ranks mapped to ids by a seeded permutation of the vocabulary."""
    ranks = torch.arange(1, VOCAB + 1, dtype=torch.float64, device="cuda")
    cdf = torch.cumsum(ranks.pow(-s), 0)
    cdf = (cdf / cdf[-1]).float()
    perm = torch.randperm(VOCAB, generator=gen, device="cuda").to(torch.int32)
    out = torch.empty(n, dtype=torch.int32, device="cuda")
    for a in range(0, n, 1 << 26):
        b = min(n, a + (1 << 26))
        u = torch.rand(b - a, generator=gen, device="cuda")
        out[a:b] = perm[torch.searchsorted(cdf, u).clamp_(max=VOCAB - 1)]
    return out


def step_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return float(np.median(times))


def encoded(ids):
    t = np.asarray(ids, dtype=np.int64)
    out = np.empty((len(t), 3), dtype=np.uint8)
    out[:, 0], out[:, 1], out[:, 2] = 0x80 | (t >> 14), (t >> 7) & 0x7F, t & 0x7F
    return out.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=256 * 1024)
    ap.add_argument("--tokens", type=int, default=2048)
    ap.add_argument("--patterns", type=int, default=100_000)
    ap.add_argument("--gram", type=int, default=13)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=64)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}), flush=True)

    gen = torch.Generator(device="cuda")
    gen.manual_seed(1234)
    n_docs, per, g = args.docs, args.tokens, args.gram
    N = n_docs * per
    tokens = zipf_ids(N, gen)
    offsets = torch.arange(n_docs + 1, dtype=torch.int64, device="cuda") * per
    # patterns: half are 13-grams of the data (each occurs), half fresh Zipf 13-grams
    half = args.patterns // 2
    docs = torch.randint(0, n_docs, (half,), generator=gen, device="cuda")
    at = torch.randint(0, per - g + 1, (half,), generator=gen, device="cuda")
    from_data = tokens[(docs * per + at)[:, None] + torch.arange(g, device="cuda")]
    fresh = zipf_ids((args.patterns - half) * g, gen).view(-1, g)
    pats = torch.cat([from_data, fresh]).cpu().numpy()
    t0 = time.perf_counter()
    ac = TokenAhoCorasick(list(pats), MatchKind.Standard)
    build_s = time.perf_counter() - t0
    print(json.dumps({"workload": {"docs": n_docs, "tokens_per_doc": per, "ids": N, "encoded_bytes": 3 * N,
                                   "patterns": len(pats), "gram": g, "build_s": round(build_s, 2)}}), flush=True)

    # ---- the encode kernel alone
    L = _capi.lib()
    buf = torch.empty(3 * N, dtype=torch.uint8, device="cuda")
    bad = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def encode():
        rc = L.acb_tokens_encode(tokens.data_ptr(), 4, N, buf.data_ptr(), bad.data_ptr(), stream)
        assert rc == _capi.ACB_OK, _capi.last_error()

    for _ in range(3):
        encode()
    launches = 50
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(launches):
        encode()
    ev1.record()
    ev1.synchronize()
    enc_s = ev0.elapsed_time(ev1) / 1e3 / launches
    assert int(bad.item()) == -1
    print(json.dumps({"encode": {"ms": round(enc_s * 1e3, 4), "algorithmic_GB_per_s": round(7 * N / enc_s / 1e9, 1),
                                 "share_of_3_35_TB_per_s": round(7 * N / enc_s / HBM_BYTES_PER_S, 3)}}), flush=True)
    del buf

    # ---- whole steps, and a sample of documents against the oracle
    m, mo, total = ac.scan_device(tokens, offsets)
    engine = ac.last_stats.get("engine")
    counts = ac.count_matches_device(tokens, offsets)
    flags = ac.is_match_device(tokens, offsets)
    rng = np.random.default_rng(7)
    sample = sorted(set(rng.integers(0, n_docs, args.sample).tolist()) | set(docs[:8].tolist()))
    # the oracle over 100 k patterns takes minutes to build: it gets the patterns whose 13 ids occur in a sampled
    # document (the others cannot match there), in id order, and its pattern ids are mapped back
    by_gram = {}
    for i, p in enumerate(pats.tolist()):
        by_gram.setdefault(tuple(p), []).append(i)
    sample_ids = {d: tokens[d * per:(d + 1) * per].cpu().numpy() for d in sample}
    subset = sorted({i for d in sample for k in range(per - g + 1) for i in by_gram.get(tuple(sample_ids[d][k:k + g].tolist()), ())})
    orc = Oracle([encoded(pats[i]) for i in subset], "Standard")
    mo_h = mo.cpu().numpy()
    for d in sample:
        want = [(subset[p], s // 3, e // 3) for p, s, e in orc.find(encoded(sample_ids[d]))]
        got = [tuple(r) for r in m[mo_h[d]:mo_h[d + 1], 1:].cpu().tolist()]
        assert got == want, f"document {d} differs from the oracle"
        assert int(counts[d]) == len(want) and bool(flags[d]) == bool(want)
    print(json.dumps({"verified": {"documents": len(sample), "total_matches": int(total), "engine": engine,
                                   "docs_with_match": int(flags.sum())}}), flush=True)
    del m, mo
    for name, fn in (("scan_device", lambda: ac.scan_device(tokens, offsets)),
                     ("count_matches_device", lambda: ac.count_matches_device(tokens, offsets)),
                     ("is_match_device", lambda: ac.is_match_device(tokens, offsets))):
        s = step_time(fn, args.reps)
        print(json.dumps({"step": name, "ms": round(s * 1e3, 3), "G_tokens_per_s": round(N / s / 1e9, 3),
                          "encoded_GB_per_s": round(3 * N / s / 1e9, 1), "encode_share": round(enc_s / s, 3),
                          "engine": ac.last_stats.get("engine")}), flush=True)

    # ---- stop sequences: find_first_stream_batch, per-feed latency
    for n_streams in (256, 4096):
        for step in (1, 64):
            feeds = 60
            ids = zipf_ids(n_streams * step * feeds, gen).view(feeds, n_streams * step)
            o = torch.arange(n_streams + 1, dtype=torch.int64, device="cuda") * step
            fb = ac.find_first_stream_batch(n_streams)
            for f in range(10):
                fb.feed_device(ids[f], o)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for f in range(10, feeds):
                out = fb.feed_device(ids[f], o)
            torch.cuda.synchronize()
            lat = (time.perf_counter() - t0) / (feeds - 10)
            print(json.dumps({"find_first_stream_batch": {"streams": n_streams, "tokens_per_feed": step,
                                                          "ms_per_feed": round(lat * 1e3, 3), "answered": int((out[:, 0] >= 0).sum())}}),
                  flush=True)


if __name__ == "__main__":
    main()
