// scan_global.cuh -- segment-parallel scan straight from the automaton image in
// global memory (the H100's 50 MB L2 holds the hot part of the table).
//
// The staged kernel (scan_staged.cuh) lives off a few hundred "hot" table rows in
// shared memory; that is the right tool when the scan spends its time near the
// root (sparse matches in text).  A dense automaton on adversarial data -- tens
// of thousands of random patterns over a small alphabet (BASELINE configs 4/5)
// -- is in a state of depth >= 3 most of the time, the hot set cannot cover it,
// and every few bytes a lane would fall out to the exact scanner while the other
// 31 wait.  For such data this kernel gives up on shared memory altogether: one
// THREAD per segment, the exact scanner (scan_core.cuh) all the way, one
// dependent L2 load per byte, and as many threads in flight as the SM holds to
// cover that latency.  Same decomposition and the same outputs as the staged
// kernel (speculated segment starts after a warm-up, SegInfo, unit counts), so
// the epilogue does not know the difference.
//
// The limit is L2 throughput for random 32-byte sectors (one per transition), not latency.
#pragma once
#include "scan_staged.cuh"

namespace acb {

template <int MODE, bool CP>
__global__ void __launch_bounds__(256)
scan_global_kernel(DevImage im, Batch B, SegPlan P, Sink out, SegInfo *seg_info) {
    const int64_t stream_lo = __ldg(B.offsets), stream_hi = __ldg(B.offsets + B.n_haystacks);
    for (int64_t seg = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; seg < P.n_segments; seg += (int64_t)gridDim.x * blockDim.x) {
        const int64_t glo = P.origin + seg * (int64_t)P.seg_bytes;
        const int64_t lo = max(glo, stream_lo), hi = min(glo + (int64_t)P.seg_bytes, stream_hi);
        if (lo >= hi) {
            // a segment outside the stream (the plan is sized from the buffer length): nothing to scan
            uint4 *dst = reinterpret_cast<uint4 *>(seg_info + seg);
            dst[0] = make_uint4(kNoState, kRoot, 0u, 0u);
            dst[1] = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint2 *>(out.unit_counts + 2 * seg) = make_uint2(0u, 0u);
            continue;
        }
        // the haystack containing lo: try the position an equal-length batch would put it at, else search
        int64_t h = P.avg_len ? (int64_t)((uint32_t)(lo - stream_lo) / (uint32_t)P.avg_len) : 0;
        if (h >= B.n_haystacks) h = B.n_haystacks - 1;
        int64_t hs = __ldg(B.offsets + h), he = __ldg(B.offsets + h + 1);
        if (!(hs <= lo && lo < he)) {
            h = find_haystack(B, lo);
            hs = __ldg(B.offsets + h);
            he = __ldg(B.offsets + h + 1);
        }
        const bool cont = hs < lo;
        const int64_t w = cont ? max(hs, lo - (int64_t)P.warm) : lo;  // the silent warm-up starts here
        PieceCtx c;
        LaneSeg L;
        L.org = w;
        L.seg = seg;
        L.lo_rel = (uint32_t)(lo - w);
        L.hi_rel = (uint32_t)(hi - w);
        L.h = (uint32_t)h;
        L.kind = cont ? kPieceWarm : kPieceNormal;
        L.spec_state = kNoState;
        L.head_count = 0;
        L.done = 0;
        c.base = B.bytes + w;
        c.at = 0;
        c.limit = (uint32_t)(he - w);
        c.stop = cont ? L.lo_rel : min(L.hi_rel, c.limit);
        c.emit_from = cont ? 0xffffffffu : 0u;  // the warm-up reports nothing
        c.state = kRoot;
        c.have = 0;
        c.last_pid = c.last_end = 0;
        c.hay = (uint32_t)h;
        c.hay_delta = (uint32_t)(w - hs);
        c.unit = (uint32_t)(2 * seg + 1);
        c.nemit = 0;
        c.cp_pos = 0;
        c.cp_cont = 0;
        HotMap none;
        none.full2hot = nullptr;
        none.hot_limit = 0;
        settle<MODE, CP>(c, L, im, B, out, seg_info, none, 0u, /*stop_hot=*/false);  // runs until the segment's summary is written
    }
}

}  // namespace acb
