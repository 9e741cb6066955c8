// capi.cu -- the C ABI (include/acb200.h): planning, kernel dispatch, ordering passes.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <cooperative_groups.h>

#include "repair.cuh"
#include "scan_staged.cuh"
#include "scan_global.cuh"
#include "scan_sieve.cuh"
#include "tokens.cuh"
#include "completions.cuh"

namespace acb {

// ---------------------------------------------------------------------------
// plain kernel: the exact scanner over whole haystacks, table in global memory
// (units = haystacks; used when no hot image is given, and as the cross-check
// of the staged + repair path in the tests)
// ---------------------------------------------------------------------------
template <int MODE, bool CP>
__global__ void __launch_bounds__(128) scan_plain_kernel(DevImage im, Batch B, Sink out) {
    for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h < B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) {
        const int64_t hs = B.offsets[h], he = B.offsets[h + 1];
        PieceCtx c;
        c.base = B.bytes + hs;
        c.at = 0;
        c.stop = c.limit = (uint32_t)(he - hs);
        c.emit_from = 0;
        c.state = kRoot;
        c.have = 0;
        c.last_pid = c.last_end = 0;
        c.hay = (uint32_t)h;
        c.hay_delta = 0;
        c.unit = (uint32_t)h;
        c.nemit = 0;
        c.cp_pos = 0;
        c.cp_cont = 0;
        exact_scan<MODE, CP>(c, im, out, false, 0, HotMap{nullptr, 0});
        out.unit_counts[h] = c.nemit;
    }
}

// ---------------------------------------------------------------------------
// profile kernel: walks a sample of the input through the dense table and
// counts state visits; the host ranks states by these counts to choose the rows
// the staged kernel keeps in shared memory (automaton.cpp: build_hot_image)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
profile_kernel(DevImage im, Batch B, uint32_t *visits, int64_t n_samples, uint32_t max_bytes, int restart_on_match) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_samples) return;
    // sample i reads max_bytes at stream position lo + i * (len / n_samples), staying inside one haystack
    const int64_t lo = B.offsets[0], hi = B.offsets[B.n_haystacks];
    if (hi <= lo) return;
    const int64_t p0 = lo + ((hi - lo) / n_samples) * i;
    const int64_t h = find_haystack(B, p0);
    const uint8_t *p = B.bytes + p0;
    uint64_t len = (uint64_t)(B.offsets[h + 1] - p0);
    if (len > max_bytes) len = max_bytes;
    uint32_t s = kRoot;
    for (uint64_t k = 0; k < len; k++) {
        const uint32_t e = __ldg(im.trans + (size_t)s * im.n_cols + __ldg(im.colmap + __ldg(p + k)));
        s = e & kStateMask;
        if (s == kDead || (restart_on_match && (e & kMatchFlag))) s = kRoot;
        atomicAdd(visits + s, 1u);
    }
}

// ---------------------------------------------------------------------------
// exclusive prefix sum u32[n] (strided) -> u64[n+1]: building blocks of the epilogue kernels
// ---------------------------------------------------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long *total) {
    __shared__ unsigned long long warp_sums[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < kScanThreads / 32; d <<= 1) {
            unsigned long long y = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += y;
        }
        if (lane < kScanThreads / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    const unsigned long long before = warp ? warp_sums[warp - 1] : 0;
    *total = warp_sums[kScanThreads / 32 - 1];
    __syncthreads();
    return before + x - v;
}

// item i = in[i * stride] (+ in[i * stride + 1] when PAIR: the two slots of a segment) for i in [0, n); one tile.
// dense != null: the items are also written there, packed (a strided source is read only once that way).
template <bool PAIR>
__device__ __forceinline__ unsigned long long scan_item(const uint32_t *in, uint32_t stride, uint64_t i) {
    if (PAIR) {
        const uint2 v = *reinterpret_cast<const uint2 *>(in + i * stride);
        return (unsigned long long)v.x + v.y;
    }
    return in[i * stride];
}

template <bool PAIR>
__device__ __forceinline__ void tile_sum_body(const uint32_t *in, uint32_t stride, uint64_t n, unsigned long long *tile_sums, uint64_t tile,
                                              uint32_t *dense) {
    const uint64_t base = tile * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    unsigned long long v = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; i++)
        if (base + i < n) {
            const unsigned long long x = scan_item<PAIR>(in, stride, base + i);
            if (dense) dense[base + i] = (uint32_t)x;
            v += x;
        }
    unsigned long long total;
    block_exclusive_scan(v, &total);
    if (threadIdx.x == 0) tile_sums[tile] = total;
}

// sum of tile_sums[0 .. tile): every block works out the start of its own tile (a few hundred values at most for a
// batch, a few thousand for a multi-gigabyte buffer) instead of waiting for one block to scan them all
__device__ __forceinline__ unsigned long long tile_prefix(const unsigned long long *tile_sums, uint64_t tile) {
    unsigned long long v = 0;
    for (uint64_t i = threadIdx.x; i < tile; i += kScanThreads) v += tile_sums[i];
    unsigned long long total;
    block_exclusive_scan(v, &total);
    return total;
}

template <bool PAIR>
__device__ __forceinline__ void tile_apply_body(const uint32_t *in, uint32_t stride, uint64_t n, const unsigned long long *tile_sums,
                                                unsigned long long *out, uint64_t tile) {
    const unsigned long long tile_start = tile_prefix(tile_sums, tile);
    const uint64_t base = tile * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    unsigned long long vals[kScanItems], v = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; i++) {
        vals[i] = base + i < n ? scan_item<PAIR>(in, stride, base + i) : 0;
        v += vals[i];
    }
    unsigned long long total;
    unsigned long long run = tile_start + block_exclusive_scan(v, &total);
#pragma unroll
    for (int i = 0; i < kScanItems; i++) {
        if (base + i < n) out[base + i] = run;
        run += vals[i];
        if (base + i + 1 == n) out[n] = run;
    }
}

// The head of dev_scratch: counters the kernels accumulate into.  Zero when a workspace is first used (the caller
// allocates it zeroed) and zero again after every scan (the epilogue's last phase resets them).
constexpr int kAccQueue = 0;    // u32 task counter of the staged kernel | u32 "some speculated segment start was wrong"
constexpr int kAccContFar = 1;  // u32 SegOut.cont_far: some match's haystack began more than kContSpan segments earlier
constexpr int kAccRaw = 2;      // raw matches emitted (also the allocation cursor of the raw buffer)
constexpr int kAccGroups = 3;   // 16-byte groups in the stream
constexpr int kAccTraps = 4;    // times a lane left the hot table
constexpr int kAccRepairs = 5;  // segment boundaries repaired
constexpr int kAccWords = 8;
// acb_any_match's and acb_find_first's dev_scratch: [0] task counter (low u32), [1] tasks skipped whole, [2] windows not scanned
constexpr int kAnyScratchWords = 3;

// totals[6] after a table walker's epilogue: which of its branches the scan took (the sieve epilogue uses
// totals[6..7] for its own sizes).  Results never depend on these; tests read them to know they reached a path.
constexpr unsigned kPathFarCp = 1u;     // code points: the prefix sum over all segments' continuation bytes
constexpr unsigned kPathSearch = 2u;    // per-haystack offsets by binary search (else the warp run-fill)
constexpr unsigned kPathRepaired = 4u;  // some speculated segment start was wrong: the repair pass ran

// ---------------------------------------------------------------------------
// everything after the table walkers in ONE cooperative kernel (grid-wide
// barriers between the phases):
//   1  per item (segment, or haystack for the plain kernel): its match count,
//      tile sums, one bit "has matches" (mask); segments: the check of every
//      speculated start against the end key of the segment before it
//   (repair, only when some check failed: then the counts again)
//   2  exclusive prefix sums, written for the items that have matches only
//   3  ordered output (+ code point fix-up)
//   4  per-haystack offsets into it, the totals, the counters reset
// The scan kernels leave one 8-byte key and one count per segment for phase 1
// to stream; phase 2 reads the mask and the counts of the non-empty items, so
// a sparse step costs little more than the launch.
// ---------------------------------------------------------------------------
struct EpilogueArgs {
    DevImage im;
    Batch B;
    SegPlan P;
    Sink out;
    SegOut seg;                // segments; seg.key == null: units are haystacks (plain kernel)
    const uint32_t *counts;    // per item: seg.count, or the plain kernel's per-haystack counts
    uint64_t n_items;
    uint8_t *masks;            // [n_items / 8 + 1]: bit i of byte j = item 8 j + i has matches (rewritten every scan)
    unsigned long long *tile_sums, *unit_offsets;  // unit_offsets: written for items with matches, and [n_items] = total
    unsigned long long *cont_tiles, *cont_cum;     // code points, only when seg.cont_far is set
    unsigned long long *totals, *acc;
    const acb_match *raw;
    const uint32_t *raw_seq, *raw_unit, *raw_aux;
    unsigned long long raw_cap;
    const uint32_t *pat_cplen;
    acb_match *out_buf;
    unsigned long long out_cap;
    unsigned long long *match_offsets;
    unsigned int *need_repair;  // zeroed with the totals; set when a speculated segment start was wrong
    int do_repair;
};

// phase 1 for one tile: thread t takes items [8 t, 8 t + 8) of the tile
__device__ __forceinline__ void count_tile(const EpilogueArgs &E, uint64_t tile, bool check, bool with_c0, unsigned int &dirty) {
    const uint64_t n = E.n_items;
    const uint64_t base = tile * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    uint32_t x[kScanItems];
    if (base + kScanItems <= n && !with_c0) {
        const uint4 a = *reinterpret_cast<const uint4 *>(E.counts + base), b = *reinterpret_cast<const uint4 *>(E.counts + base + 4);
        x[0] = a.x, x[1] = a.y, x[2] = a.z, x[3] = a.w, x[4] = b.x, x[5] = b.y, x[6] = b.z, x[7] = b.w;
    } else {
#pragma unroll
        for (int i = 0; i < kScanItems; i++) x[i] = base + i < n ? E.counts[base + i] + (with_c0 ? E.seg.count0[base + i] : 0u) : 0u;
    }
    unsigned long long v = 0;
    uint32_t bits = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; i++) {
        v += x[i];
        bits |= (x[i] != 0u) << i;
    }
    if (check && base < n) {
        // (repair.cuh has the same rule)
        uint32_t prev_end = base ? E.seg.key[base - 1].y : kNoState;
#pragma unroll
        for (int i = 0; i < kScanItems; i++)
            if (base + i < n) {
                const uint2 k = E.seg.key[base + i];
                dirty |= (base + i > 0 && k.x != kNoState && k.x != prev_end) ? 1u : 0u;
                prev_end = k.y;
            }
    }
    if (base < n) E.masks[base / kScanItems] = (uint8_t)bits;
    unsigned long long total;
    block_exclusive_scan(v, &total);
    if (threadIdx.x == 0) E.tile_sums[tile] = total;
}

// phase 2 for one tile: the offsets of the items that have matches
__device__ __forceinline__ void offsets_tile(const EpilogueArgs &E, uint64_t tile, bool with_c0) {
    const uint64_t n = E.n_items;
    const unsigned long long tile_start = tile_prefix(E.tile_sums, tile);
    const uint64_t base = tile * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    const uint32_t bits = base < n ? E.masks[base / kScanItems] : 0u;
    uint32_t x[kScanItems];
    unsigned long long v = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; i++) {
        x[i] = (bits >> i) & 1u ? E.counts[base + i] + (with_c0 ? E.seg.count0[base + i] : 0u) : 0u;
        v += x[i];
    }
    unsigned long long total;
    unsigned long long run = tile_start + block_exclusive_scan(v, &total);
#pragma unroll
    for (int i = 0; i < kScanItems; i++) {
        if ((bits >> i) & 1u) E.unit_offsets[base + i] = run;
        run += x[i];
        if (base + i + 1 == n) E.unit_offsets[n] = run;
    }
}

// phase 3: raw match i of unit u with rank r goes to unit_offsets[u] + r (segments: unit 2k + slot; slot 1 after
// slot 0, minus the matches the repair pass superseded); code point fix-up
__device__ __forceinline__ void order_body(const EpilogueArgs &E, unsigned long long raw_total, bool codepoints, bool repaired, bool far) {
    const bool segments = E.seg.key != nullptr;
    const unsigned long long n = raw_total < E.raw_cap ? raw_total : E.raw_cap;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t u = E.raw_unit[i];
        uint32_t seq = E.raw_seq[i];
        unsigned long long dst;
        if (segments) {
            const uint32_t k = u >> 1;
            if (repaired && (u & 1u)) {
                const uint32_t drop = E.seg.rest[k].drop;
                if (seq < drop) continue;  // superseded by the repair pass
                seq += E.seg.count0[k] - drop;
            }
            dst = E.unit_offsets[k] + seq;
        } else {
            dst = E.unit_offsets[u] + seq;
        }
        if (dst >= E.out_cap) continue;
        uint4 r = reinterpret_cast<const uint4 *>(E.raw)[i];  // haystack, pattern, start, end (bytes)
        if (codepoints) {
            unsigned long long cont = E.raw_aux[i];  // continuation bytes from the counting origin to the match end
            if (segments) {
                const int64_t j = u >> 1;
                const int64_t hs = E.B.offsets[r.x];
                if (hs < E.P.origin + j * (int64_t)E.P.seg_bytes) {
                    // the match's haystack began in an earlier segment: add what those segments counted
                    const int64_t j0 = (hs - E.P.origin) / (int64_t)E.P.seg_bytes;
                    if (far)
                        cont += E.cont_cum[j] - E.cont_cum[j0];
                    else
                        for (int64_t t = j0; t < j; t++) cont += E.seg.cont_tail[t];  // at most kContSpan
                }
            }
            const uint32_t end_cp = r.w - (uint32_t)cont;
            r.w = end_cp;
            r.z = end_cp - E.pat_cplen[r.y];
        }
        reinterpret_cast<uint4 *>(E.out_buf)[dst] = r;
    }
}

// phase 4: per-haystack CSR offsets into the ordered output + the totals
// (raw_total: read before the barrier in front of this phase, which resets the counter)
__device__ __forceinline__ void match_offsets_body(const EpilogueArgs &E, unsigned long long raw_total, unsigned paths) {
    const unsigned long long total = E.unit_offsets[E.n_items];
    const bool complete = raw_total <= E.raw_cap && total <= E.out_cap;
    const unsigned long long avail = total < E.out_cap ? total : E.out_cap;
    const int64_t nh = E.B.n_haystacks;
    const acb_match *out = E.out_buf;
    const bool run_fill = complete && avail <= 4 * (unsigned long long)(nh + 1);
    if (run_fill) {
        // Few matches per haystack: one pass over the records.  Record i is the first of every haystack in
        // (haystack of record i - 1, haystack of record i]; i == avail closes the list (haystacks up to nh).  The warp
        // fills those runs together, so a long run of haystacks without matches does not hold up one thread.
        const uint32_t lane = threadIdx.x & 31;
        for (unsigned long long wb = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); wb <= avail;
             wb += (unsigned long long)gridDim.x * blockDim.x) {
            const unsigned long long i = wb + lane;
            int64_t hp = 0, hc = 0;
            if (i <= avail) {
                hp = i ? (int64_t)out[i - 1].haystack : -1;
                hc = i < avail ? (int64_t)out[i].haystack : nh;
            }
            unsigned int pending = __ballot_sync(0xffffffffu, hc > hp);
            while (pending) {
                const int src = __ffs(pending) - 1;
                pending &= pending - 1;
                const int64_t a = __shfl_sync(0xffffffffu, hp, src) + 1, b = __shfl_sync(0xffffffffu, hc, src);
                const unsigned long long val = __shfl_sync(0xffffffffu, i, src);
                for (int64_t h = a + lane; h <= b; h += 32) E.match_offsets[h] = val;
            }
        }
    } else {
        // many matches per haystack (or an incomplete list, retried by the caller): binary search per haystack
        for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h <= nh; h += (int64_t)gridDim.x * blockDim.x) {
            unsigned long long lo = 0, hi = avail;  // first index whose haystack >= h
            while (lo < hi) {
                const unsigned long long mid = (lo + hi) >> 1;
                if ((int64_t)out[mid].haystack < h)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            E.match_offsets[h] = (h == nh) ? total : lo;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        // publish the totals, and leave the workspace's counters at zero for the next scan (nothing else
        // touches them in this phase): a scan needs no clearing launch in front of it
        unsigned long long *totals = E.totals, *acc = E.acc;
        totals[0] = total;
        totals[1] = complete ? 1 : 0;
        totals[2] = acc[kAccGroups];
        totals[3] = acc[kAccTraps];
        totals[4] = raw_total;
        totals[5] = acc[kAccRepairs];
        totals[6] = paths | (run_fill ? 0u : kPathSearch);
        totals[7] = 0;
        acc[kAccRaw] = acc[kAccGroups] = acc[kAccTraps] = acc[kAccRepairs] = 0;
        acc[kAccQueue] = 0;    // the scan kernel's task queue (low word) and the repair flag (high word)
        acc[kAccContFar] = 0;
    }
}

template <int MODE, bool CP>
__global__ void __launch_bounds__(kScanThreads) epilogue_kernel(EpilogueArgs E) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const bool segments = E.seg.key != nullptr;
    const uint64_t tiles = (E.n_items + kScanTile - 1) / kScanTile;
    // phase 1: counts as the scan kernel left them, and -- non-overlapping searches -- the boundary checks
    unsigned int dirty = 0;
    for (uint64_t tt = blockIdx.x; tt < tiles; tt += gridDim.x) count_tile(E, tt, E.do_repair != 0, false, dirty);
    if (E.do_repair && __any_sync(0xffffffffu, dirty) && (threadIdx.x & 31) == 0) atomicOr(E.need_repair, 1u);
    grid.sync();
    const bool repaired = E.do_repair && *reinterpret_cast<volatile unsigned int *>(E.need_repair);
    if (repaired) {
        // rare: some guess was wrong.  Redo those places exactly (into the slot-0 counts, cleared first), then count again.
        for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < E.n_items; k += (uint64_t)gridDim.x * blockDim.x)
            E.seg.count0[k] = 0;
        grid.sync();
        repair_body<MODE, CP>(E.im, E.B, E.P, E.out, E.seg, E.acc + kAccRepairs);
        grid.sync();
        for (uint64_t tt = blockIdx.x; tt < tiles; tt += gridDim.x) count_tile(E, tt, false, true, dirty);
        grid.sync();
    }
    // code points, when some haystack runs over many segments before a match: a prefix sum of the segments'
    // continuation bytes (the scan kernels and the repair pass raise the flag, before the last barrier)
    const bool far = CP && segments && *reinterpret_cast<volatile unsigned int *>(E.seg.cont_far);
    const uint64_t ctiles = far ? tiles : 0;
    if (far) {
        for (uint64_t tt = blockIdx.x; tt < ctiles; tt += gridDim.x)
            tile_sum_body<false>(E.seg.cont_tail, 1, E.n_items, E.cont_tiles, tt, nullptr);
        grid.sync();
    }
    // phase 2: exclusive prefix sums (every block derives its tile's start from the tile sums)
    for (uint64_t tt = blockIdx.x; tt < tiles + ctiles; tt += gridDim.x) {
        if (tt >= tiles)
            tile_apply_body<false>(E.seg.cont_tail, 1, E.n_items, E.cont_tiles, E.cont_cum, tt - tiles);
        else
            offsets_tile(E, tt, repaired);
    }
    grid.sync();
    // phase 3: ordered output; phase 4: per-haystack offsets into it
    const unsigned long long raw_total = *reinterpret_cast<volatile unsigned long long *>(E.acc + kAccRaw);
    order_body(E, raw_total, CP, repaired, far);
    grid.sync();
    match_offsets_body(E, raw_total, (far ? kPathFarCp : 0u) | (repaired ? kPathRepaired : 0u));
}


// ---------------------------------------------------------------------------
// Epilogue of the sieve scan (scan_sieve.cuh).  The scan leaves the OVERLAPPING
// match list as raw records tagged (task, rank in task); tasks are in stream
// order, so the ordered list needs prefix sums and one placement pass, no sort.
// Non-overlapping searches then SELECT from that list, per haystack (SURVEY.md
// 8c: "among occurrences with start >= s pick the minimum of (end, start, pid) /
// (start, pid) / (start, -end, pid)"; the list is sorted by (end, start, pid)),
// and the selected records are packed.  One cooperative launch.
// ---------------------------------------------------------------------------
struct SieveEpiArgs {
    Batch B;
    uint32_t *unit_counts;               // [n_tasks] from the scan; later [n_haystacks] selected per haystack
    uint64_t n_tasks;
    unsigned long long *tile_sums, *unit_offsets;  // unit_offsets: [n_tasks + 1]; later [n_haystacks] first record of each haystack
    const uint32_t *cont_tail;           // [n_tasks] (code points): continuation bytes in each task
    const uint32_t *hay_cont;            // [n_haystacks] (code points): continuation bytes between the start of the task a haystack starts in and the haystack
    unsigned long long *cont_tiles, *cont_cum;
    const acb_match *raw;
    const uint32_t *raw_seq, *raw_unit, *raw_aux;
    unsigned long long raw_cap;
    acb_match *ordered;                  // the overlapping list, ordered (overlapping search: the output buffer)
    acb_match *final_out;                // non-overlapping: the output buffer
    unsigned long long out_cap;
    const uint32_t *pat_cplen;
    int64_t origin;
    uint32_t task_bytes;
    uint32_t max_pat_len;
    int longest;                         // kModeLeftmost: 1 = LeftmostLongest, 0 = LeftmostFirst
    unsigned long long *totals, *acc, *match_offsets;
};

// index of the first record of `list[0 .. n)` whose haystack is >= h
__device__ __forceinline__ unsigned long long first_of_haystack(const acb_match *list, unsigned long long n, int64_t h) {
    unsigned long long lo = 0, hi = n;
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) >> 1;
        if ((int64_t)list[mid].haystack < h)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// The reference's non-overlapping iteration over ONE haystack, as a selection from its overlapping list r[0 .. n)
// (sorted by end, start, pattern).  The selected records are packed to the front (PACK = false: only counted); returns
// how many.
template <int MODE, bool PACK = true>
__device__ __forceinline__ uint32_t select_non_overlapping(acb_match *r, unsigned long long n, uint32_t max_len, int longest) {
    unsigned long long w = 0;
    uint32_t s = 0;  // the search restarts here (the end of the previous match)
    if (MODE == kModeStandard) {
        // the first occurrence, in list order, that starts at or after s
        for (unsigned long long i = 0; i < n; i++) {
            const uint4 m = reinterpret_cast<const uint4 *>(r)[i];
            if (m.z >= s) {
                if (PACK)
                    reinterpret_cast<uint4 *>(r)[w++] = m;
                else
                    w++;
                s = m.w;
            }
        }
        return (uint32_t)w;
    }
    unsigned long long i = 0;
    while (i < n) {
        bool have = false;
        uint4 best = make_uint4(0, 0, 0, 0);
        for (unsigned long long j = i; j < n; j++) {
            const uint4 m = reinterpret_cast<const uint4 *>(r)[j];
            if (have && m.w > best.z + max_len) break;  // everything from here on starts after `best` does
            if (m.z < s) continue;
            bool better = !have || m.z < best.z;
            if (have && m.z == best.z) better = longest ? (m.w > best.w || (m.w == best.w && m.y < best.y)) : (m.y < best.y);
            if (better) {
                best = m;
                have = true;
            }
        }
        if (!have) break;
        if (PACK)
            reinterpret_cast<uint4 *>(r)[w++] = best;  // w <= i: only records that can no longer be chosen are overwritten
        else
            w++;
        s = best.w;
        while (i < n && r[i].end <= s) i++;
    }
    return (uint32_t)w;
}

// phases 1-3 of the sieve epilogue: the ordered overlapping list, and totals[6] / [7] = its length / the raw records
// emitted (the caller's grid barrier publishes them)
template <bool CP>
__device__ __forceinline__ void sieve_order_list(const SieveEpiArgs &E, cooperative_groups::grid_group &grid) {
    const uint64_t tiles = (E.n_tasks + kScanTile - 1) / kScanTile;
    const uint64_t ctiles = CP ? tiles : 0;
    // phase 1 + 2: where each task's matches go (and, code points, the continuation bytes before each task)
    for (uint64_t tt = blockIdx.x; tt < tiles + ctiles; tt += gridDim.x) {
        if (tt >= tiles)
            tile_sum_body<false>(E.cont_tail, 1, E.n_tasks, E.cont_tiles, tt - tiles, nullptr);
        else
            tile_sum_body<false>(E.unit_counts, 1, E.n_tasks, E.tile_sums, tt, nullptr);
    }
    grid.sync();
    for (uint64_t tt = blockIdx.x; tt < tiles + ctiles; tt += gridDim.x) {
        if (tt >= tiles)
            tile_apply_body<false>(E.cont_tail, 1, E.n_tasks, E.cont_tiles, E.cont_cum, tt - tiles);
        else
            tile_apply_body<false>(E.unit_counts, 1, E.n_tasks, E.tile_sums, E.unit_offsets, tt);
    }
    grid.sync();
    // phase 3: the ordered overlapping list
    {
        unsigned long long n = E.acc[kAccRaw];
        if (n > E.raw_cap) n = E.raw_cap;
        for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
             i += (unsigned long long)gridDim.x * blockDim.x) {
            const uint32_t u = E.raw_unit[i];
            const unsigned long long dst = E.unit_offsets[u] + E.raw_seq[i];
            if (dst >= E.out_cap) continue;
            uint4 r = reinterpret_cast<const uint4 *>(E.raw)[i];  // haystack, pattern, start, end (bytes)
            if (CP) {
                // continuation bytes between the haystack's start and the match's end: both counts are relative to
                // the start of the task they were taken in, cont_cum carries them to a common origin
                const int64_t hs = E.B.offsets[r.x];
                const int64_t u0 = (hs - E.origin) / (int64_t)E.task_bytes;
                const unsigned long long cont = (E.cont_cum[u] + E.raw_aux[i]) - (E.cont_cum[u0] + E.hay_cont[r.x]);
                const uint32_t end_cp = r.w - (uint32_t)cont;
                r.w = end_cp;
                r.z = end_cp - E.pat_cplen[r.y];
            }
            reinterpret_cast<uint4 *>(E.ordered)[dst] = r;
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            E.totals[6] = E.unit_offsets[E.n_tasks];
            E.totals[7] = E.acc[kAccRaw];
        }
    }
}

template <int MODE, bool CP>
__global__ void __launch_bounds__(kScanThreads) sieve_epilogue_kernel(SieveEpiArgs E) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    sieve_order_list<CP>(E, grid);
    {
        if (MODE != kModeOverlap) {
            // the per-haystack selection counts start at zero (the task counts in this array were consumed by phase 2)
            for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h < E.B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) E.unit_counts[h] = 0;
        }
    }
    grid.sync();
    // (from here on unit_counts / unit_offsets are per HAYSTACK: the task-level values have been consumed)
    const unsigned long long list_total = E.totals[6];
    const unsigned long long avail = list_total < E.out_cap ? list_total : E.out_cap;
    if (list_total > E.out_cap || E.totals[7] > E.raw_cap) {
        // The buffers were too small: the ordered list has holes (stale records): nothing may be read from it, not even
        // the haystack ids for the per-haystack offsets.
        // Report how much room is needed; the caller retries.  (Every block takes this branch: totals[6..7] were
        // published before the barrier and nobody writes them again.)
        for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h <= E.B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) E.match_offsets[h] = 0;
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            const unsigned long long raw_total = E.totals[7];
            E.totals[0] = list_total;
            E.totals[1] = 0;
            E.totals[2] = E.totals[3] = E.totals[5] = 0;
            E.totals[4] = raw_total > list_total ? raw_total : list_total;
            E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
            E.acc[kAccQueue] = 0;
        }
        return;
    }
    if (MODE == kModeOverlap) {
        // per-haystack offsets into the list: the first record of every haystack is found where the haystack id changes
        // (one pass over the records; the haystacks in between, which have no matches, get the same offset)
        const int64_t nh = E.B.n_haystacks;
        if (avail == 0) {
            for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h <= nh; h += (int64_t)gridDim.x * blockDim.x) E.match_offsets[h] = h == nh ? list_total : 0;
        } else {
            for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < avail; i += (unsigned long long)gridDim.x * blockDim.x) {
                const int64_t hc = (int64_t)E.ordered[i].haystack, hp = i ? (int64_t)E.ordered[i - 1].haystack : -1;
                for (int64_t h = hp + 1; h <= hc; h++) E.match_offsets[h] = i;
                if (i + 1 == avail)
                    for (int64_t h = hc + 1; h <= nh; h++) E.match_offsets[h] = h == nh ? list_total : avail;
            }
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            const unsigned long long raw_total = E.acc[kAccRaw];
            E.totals[0] = list_total;
            E.totals[1] = (raw_total <= E.raw_cap && list_total <= E.out_cap) ? 1 : 0;
            E.totals[2] = E.totals[3] = E.totals[5] = 0;
            E.totals[4] = raw_total > list_total ? raw_total : list_total;
            E.totals[7] = 0;
            E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
            E.acc[kAccQueue] = 0;
        }
        return;
    }
    // phase 4: per haystack, select the non-overlapping matches and pack them to the front of the haystack's stretch.
    // A haystack's stretch starts where the haystack id changes: the thread that sees the change owns it.  (Haystacks
    // without matches keep the zero count written in phase 3.)
    const uint64_t n_hay = (uint64_t)E.B.n_haystacks;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < avail; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t hc = E.ordered[i].haystack;
        if (i && E.ordered[i - 1].haystack == hc) continue;
        unsigned long long hi = i + 1;
        while (hi < avail && E.ordered[hi].haystack == hc) hi++;
        E.unit_offsets[hc] = i;
        E.unit_counts[hc] = select_non_overlapping<MODE>(E.ordered + i, hi - i, E.max_pat_len, E.longest);
    }
    grid.sync();
    // phase 5 + 6: per-haystack offsets into the output
    const uint64_t htiles = (n_hay + kScanTile - 1) / kScanTile;
    for (uint64_t tt = blockIdx.x; tt < htiles; tt += gridDim.x) tile_sum_body<false>(E.unit_counts, 1, n_hay, E.tile_sums, tt, nullptr);
    grid.sync();
    for (uint64_t tt = blockIdx.x; tt < htiles; tt += gridDim.x) tile_apply_body<false>(E.unit_counts, 1, n_hay, E.tile_sums, E.match_offsets, tt);
    grid.sync();
    // phase 7: pack
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < avail; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint4 r = reinterpret_cast<const uint4 *>(E.ordered)[i];
        const unsigned long long k = i - E.unit_offsets[r.x];
        if (k < E.unit_counts[r.x]) {
            const unsigned long long dst = E.match_offsets[r.x] + k;
            if (dst < E.out_cap) reinterpret_cast<uint4 *>(E.final_out)[dst] = r;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const unsigned long long raw_total = E.acc[kAccRaw];
        const unsigned long long total = n_hay ? E.match_offsets[n_hay] : 0;
        E.totals[0] = total;
        E.totals[1] = (raw_total <= E.raw_cap && list_total <= E.out_cap) ? 1 : 0;
        E.totals[2] = E.totals[3] = E.totals[5] = 0;
        E.totals[4] = raw_total > list_total ? raw_total : list_total;  // room the overlapping list needs
        E.totals[7] = 0;
        E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
        E.acc[kAccQueue] = 0;
    }
}

// ---------------------------------------------------------------------------
// Non-overlapping COUNTS (acb_count_non_overlapping, acb_count_rows).  The serial selection restarts at the end s of
// every match it picks, and what it picks next depends on s alone:
//   NEXT(s) = the serial inner loop of select_non_overlapping started at the first record whose end is after s --
//             Standard: the first record with start >= s; leftmost: the best such record, with the look-ahead break.
// NEXT(s) has a higher index than every record ending at or before s.  Give record i the successor NEXT(end_i): the
// selected matches are the chain NEXT(0), NEXT(end of that), ..., and the count is its length, found by pointer
// jumping over (next, rank) pairs in ceil(log2(stretch)) rounds -- a few grid barriers instead of one thread walking
// the whole stretch.  A stretch of at most ACB_LONG_STRETCH records is still counted by one thread (the serial loop is
// faster than the barriers there).
// ---------------------------------------------------------------------------
constexpr uint32_t kNoNext = 0xffffffffu;   // end of a chain
constexpr uint32_t kLongMark = 0xffffffffu; // unit_counts[h]: haystack h's stretch takes the parallel path

struct SelRec {
    long long pid, start, end;
};
__device__ __forceinline__ SelRec sel_rec(const acb_match *r, unsigned long long j) {
    const uint4 m = reinterpret_cast<const uint4 *>(r)[j];
    return {(long long)m.y, (long long)m.z, (long long)m.w};
}
__device__ __forceinline__ SelRec sel_rec(const long long *rows, unsigned long long j) {  // (haystack, pattern, start, end)
    return {rows[4 * j + 1], rows[4 * j + 2], rows[4 * j + 3]};
}

// NEXT(s) in r[0 .. n), sorted by (end, start, pattern); n = none
template <int MODE, class T>
__device__ __forceinline__ unsigned long long next_selected(const T *r, unsigned long long n, long long s, long long max_len, int longest) {
    unsigned long long lo = 0, hi = n;  // the first record whose end is after s
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (sel_rec(r, mid).end <= s)
            lo = mid + 1;
        else
            hi = mid;
    }
    if (MODE == kModeStandard) {
        for (unsigned long long j = lo; j < n; j++)
            if (sel_rec(r, j).start >= s) return j;
        return n;
    }
    bool have = false;
    SelRec best = {0, 0, 0};
    unsigned long long at = n;
    for (unsigned long long j = lo; j < n; j++) {
        const SelRec m = sel_rec(r, j);
        if (have && m.end > best.start + max_len) break;  // everything from here on starts after `best` does
        if (m.start < s) continue;
        bool better = !have || m.start < best.start;
        if (have && m.start == best.start) better = longest ? (m.end > best.end || (m.end == best.end && m.pid < best.pid)) : (m.pid < best.pid);
        if (better) {
            best = m;
            at = j;
            have = true;
        }
    }
    return at;
}

// one round of pointer jumping for record i: pairs[i] = (next, rank) -- rank = records on the chain from i on that
// the rounds so far have summed; half `src` holds the current pairs, the other half gets the next ones
__device__ __forceinline__ void jump_pair(uint4 *pairs, unsigned long long i, int src) {
    const uint4 p = pairs[i];
    uint32_t nx = src ? p.z : p.x, rk = src ? p.w : p.y;
    if (nx != kNoNext) {
        const uint4 q = pairs[nx];
        rk += src ? q.w : q.y;
        nx = src ? q.z : q.x;
    }
    if (src)
        reinterpret_cast<uint2 *>(pairs + i)[0] = make_uint2(nx, rk);
    else
        reinterpret_cast<uint2 *>(pairs + i)[1] = make_uint2(nx, rk);
}

__device__ __forceinline__ uint32_t ceil_log2(unsigned long long x) { return x <= 1 ? 0u : 64u - (uint32_t)__clzll(x - 1); }

// a block's sum into *dst (every thread of the block calls it)
__device__ __forceinline__ void block_add(unsigned long long *dst, unsigned long long v) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, v);
}

// one past the last record of the stretch (the records of one haystack) that starts at list[i]: galloping, then binary
// search (a long stretch is not walked by one thread)
__device__ __forceinline__ unsigned long long stretch_end(const acb_match *list, unsigned long long i, unsigned long long avail) {
    const uint32_t hc = list[i].haystack;
    unsigned long long a = i + 1, step = 1;  // list[a - 1] is in the stretch
    for (;;) {
        const unsigned long long b = a + step - 1;
        if (b >= avail || list[b].haystack != hc) break;
        a = b + 1;
        step <<= 1;
    }
    unsigned long long hi = a + step - 1 < avail ? a + step - 1 : avail;
    while (a < hi) {
        const unsigned long long mid = (a + hi) >> 1;
        if (list[mid].haystack == hc)
            a = mid + 1;
        else
            hi = mid;
    }
    return a;
}

// The count variant of sieve_epilogue_kernel (MODE kModeStandard / kModeLeftmost, no code points): phases 1-3 place
// the overlapping list (from E.raw = dev_raw into E.ordered = dev_out), phase 4 counts each haystack's selection
// without packing it, straight into counts[h].  Stretches longer than ACB_LONG_STRETCH are counted by the whole grid
// (successors, then pointer jumping over (next, rank) pairs kept in dev_raw, which phase 3 has consumed: 16 bytes per
// record are two pairs, double-buffered).  totals[2] = haystacks counted that way; during the launch totals[3] sums the
// counts and totals[5] holds the longest such stretch.
template <int MODE>
__global__ void __launch_bounds__(kScanThreads) sieve_count_epilogue_kernel(SieveEpiArgs E, unsigned long long *counts) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    if (blockIdx.x == 0 && threadIdx.x == 0) E.totals[2] = E.totals[3] = E.totals[5] = 0;  // (read only after phase 4's barrier)
    sieve_order_list<false>(E, grid);
    for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h < E.B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) counts[h] = 0;
    grid.sync();
    const unsigned long long list_total = E.totals[6];
    const unsigned long long raw_total = E.totals[7];
    auto finish = [&](bool complete) {
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            E.totals[0] = complete ? E.totals[3] : list_total;
            E.totals[1] = complete ? 1 : 0;
            E.totals[3] = E.totals[5] = E.totals[7] = 0;
            E.totals[4] = raw_total > list_total ? raw_total : list_total;  // room the overlapping list needs
            E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
            E.acc[kAccQueue] = 0;
        }
    };
    if (list_total > E.out_cap || raw_total > E.raw_cap) {
        finish(false);  // the list has holes: every count stays zero, the caller retries with the room reported
        return;
    }
    const unsigned long long avail = list_total;
    const acb_match *const list = E.ordered;
    uint4 *const pairs = reinterpret_cast<uint4 *>(const_cast<acb_match *>(E.raw));
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    // phase 4: the thread that sees a haystack's first record owns its stretch
    unsigned long long sum = 0;
    for (unsigned long long i = first_i; i < avail; i += stride) {
        const uint32_t hc = list[i].haystack;
        if (i && list[i - 1].haystack == hc) continue;
        const unsigned long long a = stretch_end(list, i, avail);
        const unsigned long long len = a - i;
        if (len <= ACB_LONG_STRETCH) {
            const uint32_t c = select_non_overlapping<MODE, false>(const_cast<acb_match *>(list) + i, len, E.max_pat_len, E.longest);
            counts[hc] = c;
            E.unit_counts[hc] = 0;
            sum += c;
        } else {
            E.unit_counts[hc] = kLongMark;
            E.unit_offsets[hc] = i;
            counts[hc] = a;  // (the stretch's end, until its count replaces it)
            atomicAdd(E.totals + 2, 1ull);
            atomicMax(E.totals + 5, len);
        }
    }
    block_add(E.totals + 3, sum);
    grid.sync();
    if (E.totals[2]) {
        // successors: absolute list indices (a list of 2^32 records would not fit the device's memory twice)
        for (unsigned long long i = first_i; i < avail; i += stride) {
            const uint32_t hc = list[i].haystack;
            if (E.unit_counts[hc] != kLongMark) continue;
            const unsigned long long lo = E.unit_offsets[hc], n = counts[hc] - lo;
            const unsigned long long nx = next_selected<MODE>(list + lo, n, (long long)list[i].end, E.max_pat_len, E.longest);
            reinterpret_cast<uint2 *>(pairs + i)[0] = make_uint2(nx == n ? kNoNext : (uint32_t)(lo + nx), 1u);
        }
        grid.sync();
        const uint32_t rounds = ceil_log2(E.totals[5]);
        for (uint32_t r = 0; r < rounds; r++) {
            for (unsigned long long i = first_i; i < avail; i += stride)
                if (E.unit_counts[list[i].haystack] == kLongMark) jump_pair(pairs, i, (int)(r & 1));
            grid.sync();
        }
        // the count: the rank of the chain's head, NEXT(0)
        sum = 0;
        for (unsigned long long i = first_i; i < avail; i += stride) {
            const uint32_t hc = list[i].haystack;
            if (E.unit_counts[hc] != kLongMark || (i && list[i - 1].haystack == hc)) continue;
            const unsigned long long n = counts[hc] - i;
            const unsigned long long head = next_selected<MODE>(list + i, n, 0, E.max_pat_len, E.longest);
            const uint4 p = pairs[i + head];  // (head < n: the stretch has a record, so the selection picks one)
            const uint32_t c = (rounds & 1) ? p.w : p.y;
            counts[hc] = c;
            sum += c;
        }
        block_add(E.totals + 3, sum);
        grid.sync();
    }
    finish(true);
}

// Phase 4 of the pattern and hits epilogues, over the complete ordered list E.ordered[0 .. avail): each haystack's
// selection, found and left in place.  unit_offsets[h] = the first record of h's stretch.  A stretch of at most
// ACB_LONG_STRETCH records is selected by one thread and packed to its front (unit_counts[h] = how many; MODE
// kModeOverlap selects every record).  A longer one (unit_counts[h] = kLongMark, match_offsets[h] = its end) gets
// successors and pointer jumping as in the count variant, and MARKS its selection, the chain head = NEXT(0), NEXT(head),
// ...: mark[head] is set before the rounds, and in round k every marked record i also marks its round-k successor
// J_k(i) = NEXT^(2^k)(i), which it reads anyway.  After round k every NEXT^m(head) with m < 2^(k+1) is marked, so
// ceil(log2(stretch)) rounds mark the whole chain.  Only chain records are ever marked (the chain is closed under J_k),
// so a mark another thread sets in the same round and this one already sees only marks a chain record sooner: the race
// needs no barrier.  The marks live in raw_seq (u32 per record, consumed by phase 3); the pairs' rank words are computed
// and unused.  (kModeOverlap: a long stretch is selected whole and nothing is marked.)  totals[2] = the long stretches,
// totals[5] = the longest.  Ends with a grid barrier.
template <int MODE>
__device__ __forceinline__ void select_stretches(const SieveEpiArgs &E, cooperative_groups::grid_group &grid, unsigned long long avail) {
    acb_match *const list = E.ordered;
    uint4 *const pairs = reinterpret_cast<uint4 *>(const_cast<acb_match *>(E.raw));
    uint32_t *const mark = const_cast<uint32_t *>(E.raw_seq);
    unsigned long long *const ends = E.match_offsets;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    // the thread that sees a haystack's first record owns its stretch
    for (unsigned long long i = first_i; i < avail; i += stride) {
        const uint32_t hc = list[i].haystack;
        if (i && list[i - 1].haystack == hc) continue;
        const unsigned long long a = stretch_end(list, i, avail);
        const unsigned long long len = a - i;
        E.unit_offsets[hc] = i;
        if (len <= ACB_LONG_STRETCH) {
            E.unit_counts[hc] = MODE == kModeOverlap ? (uint32_t)len : select_non_overlapping<MODE>(list + i, len, E.max_pat_len, E.longest);
        } else {
            E.unit_counts[hc] = kLongMark;
            ends[hc] = a;
            // the chain's head, relative, in the second half of the first record's pair until the successors are written
            if (MODE != kModeOverlap) pairs[i].z = (uint32_t)next_selected<MODE>(list + i, len, 0, E.max_pat_len, E.longest);
            atomicAdd(E.totals + 2, 1ull);
            atomicMax(E.totals + 5, len);
        }
    }
    grid.sync();
    if (MODE != kModeOverlap && E.totals[2]) {
        for (unsigned long long i = first_i; i < avail; i += stride) {
            const uint32_t hc = list[i].haystack;
            if (E.unit_counts[hc] != kLongMark) continue;
            const unsigned long long lo = E.unit_offsets[hc], n = ends[hc] - lo;
            const unsigned long long nx = next_selected<MODE>(list + lo, n, (long long)list[i].end, E.max_pat_len, E.longest);
            reinterpret_cast<uint2 *>(pairs + i)[0] = make_uint2(nx == n ? kNoNext : (uint32_t)(lo + nx), 1u);
            mark[i] = i == lo + pairs[lo].z ? 1u : 0u;
        }
        grid.sync();
        const uint32_t rounds = ceil_log2(E.totals[5]);
        for (uint32_t r = 0; r < rounds; r++) {
            const int src = (int)(r & 1);
            for (unsigned long long i = first_i; i < avail; i += stride) {
                if (E.unit_counts[list[i].haystack] != kLongMark) continue;
                const uint32_t j = src ? pairs[i].z : pairs[i].x;  // J_r(i)
                if (j != kNoNext && mark[i]) mark[j] = 1u;
                jump_pair(pairs, i, src);
            }
            grid.sync();
        }
    }
}

// The per-pattern variant of sieve_count_epilogue_kernel (acb_pattern_counts_non_overlapping): phases 1-3 place the
// overlapping list, select_stretches finds each haystack's selection, and a last pass over the list adds the pid of
// every selected record to pattern_counts[pid].  totals[0] sums the selected records during the launch, totals[2] =
// haystacks selected on the grid, totals[5] = the longest such stretch; ws->dev_match_offsets holds each long stretch's
// end.  Nothing is added when the list did not fit.
template <int MODE>
__global__ void __launch_bounds__(kScanThreads) sieve_pattern_epilogue_kernel(SieveEpiArgs E, unsigned long long *pattern_counts) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    if (blockIdx.x == 0 && threadIdx.x == 0) E.totals[0] = E.totals[2] = E.totals[5] = 0;  // (read and added to only after later barriers)
    sieve_order_list<false>(E, grid);
    grid.sync();
    const unsigned long long list_total = E.totals[6];
    const unsigned long long raw_total = E.totals[7];
    const bool complete = list_total <= E.out_cap && raw_total <= E.raw_cap;  // (else the list has holes: nothing is added)
    if (complete) {
        const unsigned long long avail = list_total;
        select_stretches<MODE>(E, grid, avail);
        const acb_match *const list = E.ordered;
        const uint32_t *const mark = E.raw_seq;
        const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
        const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
        // the selected records' pids: whole warps step through the list together, so equal pids of a step add once
        unsigned long long sum = 0;
        for (unsigned long long w = first_i & ~31ull; w < avail; w += stride) {
            const unsigned long long i = w + (threadIdx.x & 31u);
            bool sel = false;
            uint32_t pid = 0;
            if (i < avail) {
                const uint4 r = reinterpret_cast<const uint4 *>(list)[i];  // haystack, pattern, start, end
                const uint32_t c = E.unit_counts[r.x];
                sel = c == kLongMark ? mark[i] != 0 : i - E.unit_offsets[r.x] < c;
                pid = r.y;
            }
            const uint32_t act = __ballot_sync(0xffffffffu, sel);
            if (sel) add_per_pattern(pattern_counts, act, pid);
            sum += sel ? 1u : 0u;
        }
        block_add(E.totals, sum);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (!complete) E.totals[0] = list_total;  // the caller retries with the room reported
        E.totals[1] = complete ? 1 : 0;
        E.totals[3] = E.totals[5] = E.totals[7] = 0;
        E.totals[4] = raw_total > list_total ? raw_total : list_total;  // room the overlapping list needs
        E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
        E.acc[kAccQueue] = 0;
    }
}

// The match-mask variant (acb_match_mask_non_overlapping): phases 1-3 place the overlapping list, select_stretches
// finds each haystack's selection as in the pattern epilogue, and every selected record ORs the bits of its bytes,
// bit_base + offsets[h] + [start, end), into `mask`.  totals[0] sums the selected records during the launch, totals[2]
// = haystacks selected on the grid, totals[5] = the longest such stretch.  Nothing is OR-ed when the list did not fit.
template <int MODE>
__global__ void __launch_bounds__(kScanThreads) sieve_mask_epilogue_kernel(SieveEpiArgs E, uint32_t *mask, unsigned long long bit_base) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    if (blockIdx.x == 0 && threadIdx.x == 0) E.totals[0] = E.totals[2] = E.totals[5] = 0;  // (read and added to only after later barriers)
    sieve_order_list<false>(E, grid);
    grid.sync();
    const unsigned long long list_total = E.totals[6];
    const unsigned long long raw_total = E.totals[7];
    const bool complete = list_total <= E.out_cap && raw_total <= E.raw_cap;  // (else the list has holes: nothing is OR-ed)
    if (complete) {
        const unsigned long long avail = list_total;
        select_stretches<MODE>(E, grid, avail);
        const uint32_t *const mark = E.raw_seq;
        unsigned long long sum = 0;
        for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < avail;
             i += (unsigned long long)gridDim.x * blockDim.x) {
            const uint4 r = reinterpret_cast<const uint4 *>(E.ordered)[i];  // haystack, pattern, start, end
            const uint32_t c = E.unit_counts[r.x];
            if (c == kLongMark ? mark[i] != 0 : i - E.unit_offsets[r.x] < c) {
                or_bits(mask, bit_base + (unsigned long long)E.B.offsets[r.x] + r.z, r.w - r.z);
                sum++;
            }
        }
        block_add(E.totals, sum);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (!complete) E.totals[0] = list_total;  // the caller retries with the room reported
        E.totals[1] = complete ? 1 : 0;
        E.totals[3] = E.totals[5] = E.totals[7] = 0;
        E.totals[4] = raw_total > list_total ? raw_total : list_total;  // room the overlapping list needs
        E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
        E.acc[kAccQueue] = 0;
    }
}

// acb_mask_rows: rows (haystack, pattern, start, end) of T = int32 (acb_match) or int64, haystack-relative; each ORs
// bits bit_base + offsets[h] + [start, end).  Rows naming a haystack outside [0, n_haystacks) or an empty or negative
// span are skipped.
template <class T>
__global__ void mask_rows_kernel(const T *rows, unsigned long long n, const int64_t *offsets, int64_t n_haystacks, uint32_t *mask,
                                 unsigned long long bit_base) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const long long h = (long long)rows[4 * i], s = (long long)rows[4 * i + 2], e = (long long)rows[4 * i + 3];
        if (h < 0 || h >= n_haystacks || s < 0 || e <= s) continue;
        or_bits(mask, bit_base + (unsigned long long)(offsets[h] + s), (uint32_t)(e - s));
    }
}

// acb_mask_unpack: out[i] = bit bit_base + stride * i of mask, 16 outputs per thread (one 16-byte store when aligned)
__global__ void __launch_bounds__(256) mask_unpack_kernel(const uint32_t *mask, unsigned long long bit_base, unsigned long long stride,
                                                          unsigned long long n, uint8_t *out) {
    for (unsigned long long i0 = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) * 16; i0 < n;
         i0 += (unsigned long long)gridDim.x * blockDim.x * 16) {
        uint32_t v[4] = {0, 0, 0, 0};
        const unsigned long long m = n - i0 < 16 ? n - i0 : 16;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            if ((unsigned long long)k < m) {
                const unsigned long long b = bit_base + stride * (i0 + k);
                v[k >> 2] |= ((__ldg(mask + (b >> 5)) >> (b & 31u)) & 1u) << (8 * (k & 3));
            }
        }
        if (m == 16 && (reinterpret_cast<uintptr_t>(out + i0) & 15u) == 0) {
            *reinterpret_cast<uint4 *>(out + i0) = make_uint4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int k = 0; k < 16; k++)
                if ((unsigned long long)k < m) out[i0 + k] = (uint8_t)(v[k >> 2] >> (8 * (k & 3)));
        }
    }
}

// ---------------------------------------------------------------------------
// HITS (acb_pattern_hits): each haystack's distinct patterns, with how many of its selected records have each one.
// ---------------------------------------------------------------------------
constexpr uint32_t kHitsSmemKeys = 1024;  // per-warp shared sort buffer: 4 KiB, 32 KiB per block (4 blocks per SM still fit)

// u32 words of one counter row: n_patterns counters (padded to an even count), then u64 [haystack, nonzero counters in
// tile 0, tile 1, ...] (tiles of kScanTile counters)
__host__ __device__ __forceinline__ unsigned long long hit_row_words(unsigned long long n_patterns) {
    return (n_patterns + 1) / 2 * 2 + 2 + 2 * ((n_patterns + kScanTile - 1) / kScanTile);
}

// rows[key] += the lanes of `act` that hold key: one atomic per distinct key (called by exactly the lanes of act)
__device__ __forceinline__ void add_to_row(uint32_t *rows, uint32_t act, unsigned long long key) {
    const uint32_t peers = __match_any_sync(act, key);
    if ((threadIdx.x & 31u) == (uint32_t)__ffs(peers) - 1u) atomicAdd(rows + key, (uint32_t)__popc(peers));
}

// the warp's 32 values, ascending across the lanes (bitonic network over shuffles)
__device__ __forceinline__ uint32_t warp_sort32(uint32_t x) {
    const uint32_t lane = threadIdx.x & 31u;
#pragma unroll
    for (uint32_t k = 2; k <= 32; k <<= 1)
#pragma unroll
        for (uint32_t j = k >> 1; j; j >>= 1) {
            const uint32_t y = __shfl_xor_sync(0xffffffffu, x, j);
            x = (((lane & j) == 0) == ((lane & k) == 0)) ? min(x, y) : max(x, y);
        }
    return x;
}

// The hits of a selection of at most 32 records sel[0 .. n): the pids sorted in registers, runs found with a ballot;
// hit k = (h, pid, run length, 0) goes to out[k].  -> how many hits.
__device__ __forceinline__ uint32_t warp_hits32(const acb_match *sel, uint32_t n, uint32_t h, uint4 *out) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t k = warp_sort32(lane < n ? sel[lane].pattern : 0xffffffffu);
    const uint32_t prev = __shfl_up_sync(0xffffffffu, k, 1);
    const bool head = lane < n && (lane == 0 || prev != k);
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    if (head) {
        const uint32_t later = heads & ~((2u << lane) - 1u);
        const uint32_t end = later ? (uint32_t)__ffs(later) - 1u : n;
        out[__popc(heads & ((1u << lane) - 1u))] = make_uint4(h, k, end - lane, 0u);
    }
    return (uint32_t)__popc(heads);
}

// keys[0 .. n) ascending, by one warp (shared or global memory): the bitonic network in its flip form, where every
// comparator puts the smaller key first, so positions past n act as +infinity and their comparators are skipped
__device__ __forceinline__ void warp_sort_keys(uint32_t *keys, uint32_t n) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t half = (n <= 1 ? 1u : 1u << (32 - __clz(n - 1))) >> 1;  // comparators per step
    for (uint32_t k = 2; k <= 2 * half; k <<= 1) {
        for (uint32_t j = k >> 1; j; j >>= 1) {
            for (uint32_t p = lane; p < half; p += 32) {
                const uint32_t a = ((p & ~(j - 1)) << 1) | (p & (j - 1));  // (bit j of a is clear)
                const uint32_t b = j == k >> 1 ? a ^ (k - 1) : a ^ j;
                if (b < n) {
                    const uint32_t x = keys[a], y = keys[b];
                    if (x > y) {
                        keys[a] = y;
                        keys[b] = x;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// the runs of sorted keys[0 .. n) as hits (h, key, run length, 0) at out[0 ..), by one warp -> how many
__device__ __forceinline__ uint32_t warp_runs(const uint32_t *keys, uint32_t n, uint32_t h, uint4 *out) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t d = 0;
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t j = base + lane;
        const uint32_t k = j < n ? keys[j] : 0u;
        const bool head = j < n && (j == 0 || keys[j - 1] != k);
        const uint32_t heads = __ballot_sync(0xffffffffu, head);
        if (head) {
            uint32_t lo = j + 1, hi = n;  // the run's end: the first key above k
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (keys[mid] == k)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            out[d + __popc(heads & ((1u << lane) - 1u))] = make_uint4(h, k, lo - j, 0u);
        }
        d += (uint32_t)__popc(heads);
    }
    return d;
}

// The hits epilogue (acb_pattern_hits; MODE kModeStandard / kModeLeftmost, or kModeOverlap for the overlapping search):
// phases 1-3 place the overlapping list, select_stretches finds each haystack's selection (kModeOverlap: all of it),
// and each haystack's selected pids become its d_h hits (pid, count), pids ascending, staged at the haystack's stretch
// offset in dev_raw (d_h <= the stretch's records, so the slices never overlap; the pairs there are dead by then).
//   short stretch: one warp per haystack.  Up to 32 pids are sorted in registers; up to kHitsSmemKeys in the warp's
//     shared buffer; up to ACB_LONG_STRETCH in the stretch's slice of raw_seq (consumed by phase 3, unmarked for a short
//     stretch, in L2); then run-length encoded.
//   long stretch: a dense counter row in `rows` (slot from totals[3], only the used rows are zeroed).  Whole warps add
//     the selected pids to it, as the pattern epilogue's last pass does, and a prefix over each row's nonzero counters
//     (tiles, as tile_sum_body / tile_apply_body) stages its hits in pid order, without a sort.
// Then phases 5-6 of the list epilogue give the per-haystack offsets, and the hits are packed from dev_raw into dev_out
// (where the ordered list lived).  totals[2] = long stretches, [3] = rows used, [5] = row words needed.
template <int MODE>
__global__ void __launch_bounds__(kScanThreads) sieve_hits_epilogue_kernel(SieveEpiArgs E, uint32_t *rows, unsigned long long row_words,
                                                                           uint32_t n_patterns) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ uint32_t sort_keys[kScanThreads / 32][kHitsSmemKeys];
    if (blockIdx.x == 0 && threadIdx.x == 0) E.totals[2] = E.totals[3] = E.totals[5] = 0;  // (read and added to only after later barriers)
    sieve_order_list<false>(E, grid);
    const int64_t nh = E.B.n_haystacks;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    // haystacks without records have no hits (the task counts in this array were consumed by phase 2)
    for (int64_t h = (int64_t)first_i; h < nh; h += (int64_t)stride) E.unit_counts[h] = 0;
    grid.sync();
    const unsigned long long list_total = E.totals[6];
    const unsigned long long raw_total = E.totals[7];
    const unsigned long long rw = hit_row_words(n_patterns);
    // (else the list has holes: nothing is written, the caller retries with the room reported)
    bool complete = list_total <= E.out_cap && list_total <= E.raw_cap && raw_total <= E.raw_cap;
    unsigned long long n_long = 0;
    if (complete) {
        select_stretches<MODE>(E, grid, list_total);
        n_long = E.totals[2];
        complete = n_long * rw <= row_words;
    }
    if (complete) {
        const unsigned long long avail = list_total;
        const acb_match *const list = E.ordered;
        const uint32_t *const mark = E.raw_seq;
        uint4 *const staged = reinterpret_cast<uint4 *>(const_cast<acb_match *>(E.raw));
        unsigned long long *const slot = E.match_offsets;  // a long stretch's row (its end is no longer needed)
        const uint32_t lane = threadIdx.x & 31u;
        const uint64_t tpr = ((uint64_t)n_patterns + kScanTile - 1) / kScanTile;
        auto meta = [&](unsigned long long s) { return reinterpret_cast<unsigned long long *>(rows + (s + 1) * rw - 2 - 2 * tpr); };
        if (n_long) {
            for (int64_t h = (int64_t)first_i; h < nh; h += (int64_t)stride)
                if (E.unit_counts[h] == kLongMark) {
                    const unsigned long long s = atomicAdd(E.totals + 3, 1ull);
                    slot[h] = s;
                    meta(s)[0] = (unsigned long long)h;
                }
            for (unsigned long long s = 0; s < n_long; s++)
                for (unsigned long long p = first_i; p < n_patterns; p += stride) rows[s * rw + p] = 0;
            grid.sync();
            // the long stretches' selected pids into their rows: whole warps step through the list together, so equal
            // counters of a step add once
            for (unsigned long long w = first_i & ~31ull; w < avail; w += stride) {
                const unsigned long long i = w + lane;
                bool sel = false;
                unsigned long long key = 0;
                if (i < avail) {
                    const uint4 r = reinterpret_cast<const uint4 *>(list)[i];  // haystack, pattern, start, end
                    if (E.unit_counts[r.x] == kLongMark) {
                        sel = MODE == kModeOverlap || mark[i] != 0;
                        key = slot[r.x] * rw + r.y;
                    }
                }
                const uint32_t act = __ballot_sync(0xffffffffu, sel);
                if (sel) add_to_row(rows, act, key);
            }
        }
        // the short stretches: one warp per haystack (a long stretch's kLongMark is never a short one's count)
        uint32_t *const smem_keys = sort_keys[threadIdx.x >> 5];
        for (unsigned long long h = first_i >> 5; h < (unsigned long long)nh; h += stride >> 5) {
            const uint32_t c = E.unit_counts[h];
            if (c == 0 || c == kLongMark) continue;
            const unsigned long long lo = E.unit_offsets[h];
            uint32_t d;
            if (c <= 32) {
                d = warp_hits32(list + lo, c, (uint32_t)h, staged + lo);
            } else {
                uint32_t *const keys = c <= kHitsSmemKeys ? smem_keys : const_cast<uint32_t *>(mark) + lo;
                for (uint32_t j = lane; j < c; j += 32) keys[j] = list[lo + j].pattern;
                __syncwarp();
                warp_sort_keys(keys, c);
                d = warp_runs(keys, c, (uint32_t)h, staged + lo);
                __syncwarp();  // (the shared buffer serves the warp's next haystack)
            }
            if (lane == 0) E.unit_counts[h] = d;
        }
        grid.sync();
        if (n_long) {
            // each row's nonzero counters: per tile, then each tile's start within its row, and the hits staged
            const uint64_t tiles = n_long * tpr;
            for (uint64_t tt = blockIdx.x; tt < tiles; tt += gridDim.x) {
                const uint64_t s = tt / tpr, t = tt % tpr;
                const uint32_t *const row = rows + s * rw;
                const uint64_t base = t * kScanTile + (uint64_t)threadIdx.x * kScanItems;
                unsigned long long v = 0;
#pragma unroll
                for (int i = 0; i < kScanItems; i++) v += (base + i < n_patterns && row[base + i]) ? 1u : 0u;
                unsigned long long total;
                block_exclusive_scan(v, &total);
                if (threadIdx.x == 0) meta(s)[1 + t] = total;
            }
            grid.sync();
            for (uint64_t tt = blockIdx.x; tt < tiles; tt += gridDim.x) {
                const uint64_t s = tt / tpr, t = tt % tpr;
                const uint32_t *const row = rows + s * rw;
                const unsigned long long *const m = meta(s);
                const unsigned long long hc = m[0], lo = E.unit_offsets[hc];
                const unsigned long long tile_start = tile_prefix(m + 1, t);
                const uint64_t base = t * kScanTile + (uint64_t)threadIdx.x * kScanItems;
                uint32_t vals[kScanItems];
                unsigned long long v = 0;
#pragma unroll
                for (int i = 0; i < kScanItems; i++) {
                    vals[i] = base + i < n_patterns ? row[base + i] : 0u;
                    v += vals[i] ? 1u : 0u;
                }
                unsigned long long total;
                unsigned long long at = lo + tile_start + block_exclusive_scan(v, &total);
#pragma unroll
                for (int i = 0; i < kScanItems; i++)
                    if (vals[i]) staged[at++] = make_uint4((uint32_t)hc, (uint32_t)(base + i), vals[i], 0u);
                if (t == tpr - 1 && threadIdx.x == 0) E.unit_counts[hc] = (uint32_t)(tile_start + total);
            }
            grid.sync();
        }
        // phase 5 + 6: per-haystack offsets into the output
        const uint64_t n_hay = (uint64_t)nh;
        const uint64_t htiles = (n_hay + kScanTile - 1) / kScanTile;
        for (uint64_t tt = blockIdx.x; tt < htiles; tt += gridDim.x) tile_sum_body<false>(E.unit_counts, 1, n_hay, E.tile_sums, tt, nullptr);
        grid.sync();
        for (uint64_t tt = blockIdx.x; tt < htiles; tt += gridDim.x) tile_apply_body<false>(E.unit_counts, 1, n_hay, E.tile_sums, E.match_offsets, tt);
        grid.sync();
        // pack: output o belongs to the last haystack h with match_offsets[h] <= o
        const unsigned long long n_hits = E.match_offsets[n_hay];
        for (unsigned long long o = first_i; o < n_hits; o += stride) {
            uint64_t lo = 0, hi = n_hay;  // match_offsets[lo] <= o < match_offsets[hi]
            while (hi - lo > 1) {
                const uint64_t mid = (lo + hi) >> 1;
                if (E.match_offsets[mid] <= o)
                    lo = mid;
                else
                    hi = mid;
            }
            reinterpret_cast<uint4 *>(E.final_out)[o] = staged[E.unit_offsets[lo] + (o - E.match_offsets[lo])];
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) E.totals[0] = n_hits;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (!complete) E.totals[0] = 0;
        E.totals[1] = complete ? 1 : 0;
        E.totals[3] = complete ? n_long : 0;
        E.totals[4] = raw_total > list_total ? raw_total : list_total;  // room the overlapping list needs
        E.totals[5] = n_long * rw;                                      // row words needed (once the list fits)
        E.acc[kAccRaw] = E.acc[kAccGroups] = E.acc[kAccTraps] = E.acc[kAccRepairs] = 0;
        E.acc[kAccQueue] = 0;
    }
}

// acb_count_rows: the same successors and pointer jumping over the rows of ONE haystack (int64, as
// acb_select_non_overlapping reads them), pairs in scratch (16 bytes per row).  Cooperative, one launch.
__global__ void __launch_bounds__(kScanThreads) count_rows_kernel(const long long *rows, unsigned long long n, int mode, int longest,
                                                                 long long max_len, uint4 *pairs, unsigned long long *count) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (unsigned long long i = first_i; i < n; i += stride) {
        const long long s = rows[4 * i + 3];
        const unsigned long long nx = mode == kModeStandard ? next_selected<kModeStandard>(rows, n, s, max_len, longest)
                                                            : next_selected<kModeLeftmost>(rows, n, s, max_len, longest);
        reinterpret_cast<uint2 *>(pairs + i)[0] = make_uint2(nx == n ? kNoNext : (uint32_t)nx, 1u);
    }
    grid.sync();
    const uint32_t rounds = ceil_log2(n);
    for (uint32_t r = 0; r < rounds; r++) {
        for (unsigned long long i = first_i; i < n; i += stride) jump_pair(pairs, i, (int)(r & 1));
        grid.sync();
    }
    if (first_i == 0) {
        const unsigned long long head = mode == kModeStandard ? next_selected<kModeStandard>(rows, n, 0, max_len, longest)
                                                              : next_selected<kModeLeftmost>(rows, n, 0, max_len, longest);
        const uint4 p = pairs[head];
        *count = (rounds & 1) ? p.w : p.y;
    }
}

// ---------------------------------------------------------------------------
// Multi-GPU: the block a rank contributes to the gather of the match lists --
// row 0 = (count, haystack base, complete flag, 0), then its first `cap`
// matches -- assembled by ONE launch straight from a scan's output buffers.
// ---------------------------------------------------------------------------
__global__ void pack_gather_block_kernel(const unsigned long long *totals, const acb_match *out, uint32_t hay_base, unsigned long long cap,
                                         uint4 *block) {
    const unsigned long long total = totals[0];
    const unsigned long long n = total < cap ? total : cap;
    if (blockIdx.x == 0 && threadIdx.x == 0)
        block[0] = make_uint4((uint32_t)(total > 0xffffffffull ? 0xffffffffull : total), hay_base, (uint32_t)totals[1], 0u);
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        block[1 + i] = reinterpret_cast<const uint4 *>(out)[i];
}

// ---------------------------------------------------------------------------
// The non-overlapping selection (select_non_overlapping above) for ONE haystack whose overlapping list was
// assembled by the caller from several scans (a haystack above one call's 32-bit range): rows of four int64
// (haystack, pattern, start, end), sorted by (end, start, pattern).  One thread: the selection is a chain.
// ---------------------------------------------------------------------------
__global__ void select_rows_kernel(const long long *rows, unsigned long long n, int mode, int longest, long long max_len, long long *out,
                                   unsigned long long *count) {
    if (blockIdx.x || threadIdx.x) return;
    unsigned long long w = 0;
    long long s = 0;
    auto put = [&](unsigned long long j) {
        for (int c = 0; c < 4; c++) out[4 * w + c] = rows[4 * j + c];
        w++;
    };
    if (mode == kModeStandard) {
        for (unsigned long long i = 0; i < n; i++)
            if (rows[4 * i + 2] >= s) {
                s = rows[4 * i + 3];
                put(i);
            }
    } else {
        unsigned long long i = 0;
        while (i < n) {
            bool have = false;
            unsigned long long best = 0;
            for (unsigned long long j = i; j < n; j++) {
                const long long st = rows[4 * j + 2], en = rows[4 * j + 3], pid = rows[4 * j + 1];
                if (have && en > rows[4 * best + 2] + max_len) break;
                if (st < s) continue;
                bool better = !have || st < rows[4 * best + 2];
                if (have && st == rows[4 * best + 2])
                    better = longest ? (en > rows[4 * best + 3] || (en == rows[4 * best + 3] && pid < rows[4 * best + 1])) : (pid < rows[4 * best + 1]);
                if (better) {
                    best = j;
                    have = true;
                }
            }
            if (!have) break;
            s = rows[4 * best + 3];
            put(best);
            while (i < n && rows[4 * i + 3] <= s) i++;
        }
    }
    *count = w;
}

// ---------------------------------------------------------------------------
// acb_first_rows: first-match keys (scan_sieve.cuh, FIRST) -> int64 rows (pattern, start, end), one thread per
// haystack.  LeftmostFirst keys name (start, pattern): the end is start + the pattern's length.  The other two kinds
// name (start, end): the pattern is the lowest pid of the reverse-trie node of those bytes -- the node stage 2 found --
// reached by the same walk (hash of the W bytes before the end, then one child per byte towards the start).  With
// pattern sets (first_rows_filtered_kernel) the pattern is that node's lowest pid the haystack's set admits.
// ---------------------------------------------------------------------------
// FILT: the lowest pid of the node that `row` admits (see SieveFilter)
template <bool FILT>
__device__ __forceinline__ uint32_t sieve_pid_in(const DevSieve &sv, const uint8_t *hay, uint32_t start, uint32_t end, const uint32_t *row) {
    uint32_t lo = 0, hi = 0;  // the 8 bytes ending at end, little endian (the byte at end - 1 is the top byte of lo)
    for (uint32_t k = 1; k <= 8 && k <= end - start; k++) {
        const uint32_t b = hay[end - k];
        if (k <= 4)
            lo |= b << (8 * (4 - k));
        else
            hi |= b << (8 * (8 - k));
    }
    const uint32_t klo = sv.W <= 4 ? lo >> (8u * (4u - sv.W)) : lo, khi = sv.W <= 4 ? 0u : hi >> (8u * (8u - sv.W));
    const uint32_t x = klo + khi * kMixHi;
    uint32_t s = __umulhi(x * kMulSlot, sv.ht_size), v = kSieveNoNode;
    for (;;) {
        const SieveSlot e = sv.ht[s];
        if (e.node == kSieveNoNode) break;
        if (e.key_lo == klo && e.key_hi == khi) {
            v = e.node;
            break;
        }
        s = (s + 1) & (sv.ht_size - 1);
    }
    for (uint32_t d = sv.W; v != kSieveNoNode && d < end - start; d++) {
        const uint32_t b = hay[end - 1 - d];  // the byte before the d-byte suffix
        const uint32_t first = sv.na[v].first_kid, nk = (sv.na[v].meta >> 8) & 0x1ffu;
        uint32_t l0 = 0, l1 = nk;  // first child with byte >= b
        while (l0 < l1) {
            const uint32_t mid = (l0 + l1) >> 1;
            if ((sv.na[first + mid].meta & 0xffu) < b)
                l0 = mid + 1;
            else
                l1 = mid;
        }
        v = l0 < nk && (sv.na[first + l0].meta & 0xffu) == b ? first + l0 : kSieveNoNode;
    }
    if (v == kSieveNoNode || sv.nb[v].own_cnt == 0) return 0xffffffffu;  // (a key always names a pattern)
    if (FILT) {
        for (uint32_t t = 0; t < sv.nb[v].own_cnt; t++)
            if (filter_admits(row, sv.pids[sv.nb[v].own_off + t])) return sv.pids[sv.nb[v].own_off + t];
        return 0xffffffffu;
    }
    return sv.pids[sv.nb[v].own_off];  // ascending: the lowest index among patterns with these bytes
}

__device__ uint32_t sieve_pid_of(const DevSieve &sv, const uint8_t *hay, uint32_t start, uint32_t end) {
    return sieve_pid_in<false>(sv, hay, start, end, nullptr);
}

__global__ void first_rows_kernel(DevSieve sv, const uint32_t *pat_len, Batch B, const unsigned long long *keys, long long *rows, int kind) {
    for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h < B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[h];
        long long pid = -1, start = -1, end = -1;
        if (key != ~0ull) {
            const uint32_t hi = (uint32_t)(key >> 32), lo = (uint32_t)key;
            if (kind == ACB_LEFTMOST_FIRST) {
                start = hi;
                pid = lo;
                end = start + pat_len[lo];
            } else {
                end = kind == ACB_STANDARD ? hi : 0xffffffffu - lo;
                start = kind == ACB_STANDARD ? end - (0xffffffffu - lo) : hi;
                const uint32_t p = sieve_pid_of(sv, B.bytes + B.offsets[h], (uint32_t)start, (uint32_t)end);
                pid = p == 0xffffffffu ? -1 : (long long)p;
            }
        }
        rows[3 * h] = pid;
        rows[3 * h + 1] = start;
        rows[3 * h + 2] = end;
    }
}

// acb_first_rows with pattern sets: LeftmostFirst keys already name an admitted pattern; the other kinds take the
// node's lowest admitted pid
__global__ void first_rows_filtered_kernel(DevSieve sv, const uint32_t *pat_len, Batch B, const unsigned long long *keys, long long *rows, int kind,
                                           SieveFilter F) {
    for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h < B.n_haystacks; h += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[h];
        long long pid = -1, start = -1, end = -1;
        if (key != ~0ull) {
            const uint32_t hi = (uint32_t)(key >> 32), lo = (uint32_t)key;
            if (kind == ACB_LEFTMOST_FIRST) {
                start = hi;
                pid = lo;
                end = start + pat_len[lo];
            } else {
                end = kind == ACB_STANDARD ? hi : 0xffffffffu - lo;
                start = kind == ACB_STANDARD ? end - (0xffffffffu - lo) : hi;
                const uint32_t p = sieve_pid_in<true>(sv, B.bytes + B.offsets[h], (uint32_t)start, (uint32_t)end, filter_row(F, h));
                pid = p == 0xffffffffu ? -1 : (long long)p;
            }
        }
        rows[3 * h] = pid;
        rows[3 * h + 1] = start;
        rows[3 * h + 2] = end;
    }
}

// ---------------------------------------------------------------------------
// acb_rows_to_codepoints: byte rows -> code point rows.  The stream is cut into tiles of kCpTile bytes; a warp takes
// tiles grid-stride and, for every haystack with a row that overlaps the tile before the row's end, counts the UTF-8
// continuation bytes of that overlap before the row's start and before its end, and subtracts them from the output row
// with one atomic each.  Work is the bytes before each row's end, spread over the whole grid whatever the haystacks'
// sizes.  The input rows are only read (the output starts as their copy), so no warp sees another's subtraction.
// ---------------------------------------------------------------------------
constexpr int64_t kCpTile = 16384;

__global__ void __launch_bounds__(256) rows_to_codepoints_kernel(Batch B, int64_t buf_bytes, const long long *rows, long long *cp) {
    const uint32_t lane = threadIdx.x & 31;
    // tiles cover the buffer; the stream [offsets[0], offsets[n]) is the part of it that is counted
    const int64_t stream_lo = max(__ldg(B.offsets), (int64_t)0), stream_hi = min(__ldg(B.offsets + B.n_haystacks), buf_bytes);
    const int64_t n_tiles = (buf_bytes + kCpTile - 1) / kCpTile;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n_tiles; t += n_warps) {
        const int64_t lo = max(t * kCpTile, stream_lo), hi = min((t + 1) * kCpTile, stream_hi);
        if (lo >= hi) continue;
        for (int64_t h = find_haystack(B, lo); h < B.n_haystacks; h++) {
            const int64_t hs = __ldg(B.offsets + h);
            if (hs >= hi) break;
            const int64_t start = __ldg(rows + 3 * h + 1), end = __ldg(rows + 3 * h + 2);
            if (end < 0) continue;
            const int64_t a = max(lo, hs), be = min(hi, hs + end), bs = min(hi, hs + start);
            if (be <= a) continue;
            // 16-byte chunks at aligned addresses; bytes outside [a, be) read as zero (not a continuation byte)
            const int64_t p0 = a - (int64_t)(reinterpret_cast<uintptr_t>(B.bytes + a) & 15u);
            unsigned long long ce = 0, cs = 0;
            for (int64_t p = p0 + 16 * (int64_t)lane; p < be; p += 512) {
                uint32_t w[4] = {0, 0, 0, 0};
                if (p >= a && p + 16 <= be) {
                    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(B.bytes + p));
                    w[0] = v.x, w[1] = v.y, w[2] = v.z, w[3] = v.w;
                } else {
                    for (int k = 0; k < 16; k++)
                        if (p + k >= a && p + k < be) w[k >> 2] |= (uint32_t)__ldg(B.bytes + p + k) << (8 * (k & 3));
                }
                uint32_t m = 0;  // bit k: byte k of the chunk is a continuation byte (10xxxxxx)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t f = w[j] & ~(w[j] << 1) & 0x80808080u;
                    m |= (((f >> 7) & 1u) | ((f >> 14) & 2u) | ((f >> 21) & 4u) | ((f >> 28) & 8u)) << (4 * j);
                }
                const int64_t ks = min(max(bs - p, (int64_t)0), (int64_t)16);  // bytes of the chunk before the start
                ce += __popc(m);
                cs += __popc(m & ((1u << ks) - 1u));
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) {
                ce += __shfl_xor_sync(0xffffffffu, ce, d);
                cs += __shfl_xor_sync(0xffffffffu, cs, d);
            }
            if (lane == 0) {
                if (cs) atomicAdd(reinterpret_cast<unsigned long long *>(cp + 3 * h + 1), 0ull - cs);
                if (ce) atomicAdd(reinterpret_cast<unsigned long long *>(cp + 3 * h + 2), 0ull - ce);
            }
        }
    }
}

// when the input is empty: nothing ran, publish zeros
__global__ void zero_outputs_kernel(unsigned long long *unit_offsets, unsigned long long *match_offsets, int64_t n_haystacks,
                                    unsigned long long *totals) {
    if (blockIdx.x == 0 && threadIdx.x < 8) totals[threadIdx.x] = threadIdx.x == 1 ? 1 : 0;  // no matches, complete
    for (int64_t h = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; h <= n_haystacks; h += (int64_t)gridDim.x * blockDim.x) match_offsets[h] = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) unit_offsets[0] = 0;
}

// ---------------------------------------------------------------------------
// Stream search (acb_stream_seams / acb_stream_resolve): matches in data fed in chunks.  Per stream the caller keeps a
// carry (kCarry* words) and a tail: the last min(F, max_pattern_len - 1) bytes fed.  A feed scans the caller's chunks
// as they are, and a SEAM per stream -- tail || the chunk's first min(len, max_pattern_len - 1) bytes -- for the
// matches that cross into the chunk.  The sequence a stream selects from is: every record of its seam, then its chunk's
// records that end past the seam's head (the others are in the seam too).  Both parts are sorted by (end, start,
// pattern) and the second ends after the first, so the concatenation is the overlapping list of tail || chunk.
// ---------------------------------------------------------------------------
enum : int { kCarryFed = 0, kCarryRestart = 1, kCarryTail = 2, kCarryCont = 3, kCarryWords = 4 };

__device__ __forceinline__ bool is_cont_byte(uint32_t b) { return (b & 0xC0u) == 0x80u; }

// seam_offsets[i + 1] = tail length + head length of stream i
__global__ void stream_seam_lengths_kernel(const int64_t *offsets, int64_t n, const int64_t *carry, uint32_t halo, int64_t *seam_offsets) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = offsets[i + 1] - offsets[i];
        seam_offsets[i + 1] = carry[kCarryWords * i + kCarryTail] + min(len, (int64_t)halo);
    }
}

// v[0] = 0, v[1 .. n] = inclusive prefix sums of v[1 .. n] (one block)
__global__ void __launch_bounds__(kScanThreads) stream_prefix_kernel(int64_t *v, int64_t n) {
    unsigned long long carry = 0;
    for (int64_t base = 0; base < n; base += kScanThreads) {
        const int64_t i = base + threadIdx.x;
        const unsigned long long x = i < n ? (unsigned long long)v[i + 1] : 0ull;
        unsigned long long total;
        const unsigned long long before = block_exclusive_scan(x, &total);
        if (i < n) v[i + 1] = (int64_t)(carry + before + x);
        carry += total;
    }
    if (threadIdx.x == 0) v[0] = 0;
}

// one warp per stream: seam i = tail || head at seam_offsets[i]
__global__ void stream_seam_fill_kernel(const uint8_t *bytes, const int64_t *offsets, int64_t n, const int64_t *carry, const uint8_t *tail,
                                        uint32_t halo, const int64_t *seam_offsets, uint8_t *seam) {
    const uint32_t lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int64_t t = carry[kCarryWords * i + kCarryTail], s0 = seam_offsets[i], len = seam_offsets[i + 1] - s0;
        const uint8_t *src_tail = tail + (uint64_t)i * halo, *src_head = bytes + offsets[i];
        for (int64_t k = lane; k < len; k += 32) seam[s0 + k] = k < t ? src_tail[k] : src_head[k - t];
    }
}

// The records stream i selects from (see above), with absolute positions.
struct StreamView {
    const uint4 *seam, *chunk;
    unsigned long long ns;     // seam records; then the chunk's, from its first that ends past the head
    long long seam_base, chunk_base;
};
__device__ __forceinline__ SelRec sel_rec(const StreamView *v, unsigned long long j) {
    const bool in_seam = j < v->ns;
    const uint4 m = in_seam ? v->seam[j] : v->chunk[j - v->ns];
    const long long base = in_seam ? v->seam_base : v->chunk_base;
    return {(long long)m.y, base + (long long)m.z, base + (long long)m.w};
}

// the first record of r[lo .. hi) that ends after `after`
__device__ __forceinline__ unsigned long long first_end_after(const uint4 *r, unsigned long long lo, unsigned long long hi, uint32_t after) {
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) >> 1;
        if (r[mid].w <= after)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

struct StreamArgs {
    Batch B;                        // the chunks: one haystack per stream
    int64_t *carry;                 // [n][kCarryWords]
    uint8_t *tail;                  // [n][halo]
    const uint8_t *last;            // [n] or null
    const uint8_t *seam;
    const int64_t *seam_offsets;    // [n + 1]
    const uint4 *seam_list, *chunk_list;
    const unsigned long long *seam_mo, *chunk_mo;  // [n + 1] each
    long long *staged;              // rows (stream, pattern, start, end) of stream i from seam_mo[i] + chunk_mo[i] on
    long long *cont_rows;           // [n][3] (0, x, x): x = chunk bytes before the new tail (code points)
    long long *cont_cp;             // [n][3] the same after acb_rows_to_codepoints
    int64_t *row_offsets;           // [n + 1]
    long long *rows;                // the released rows, packed
    unsigned long long *stats;      // [0] records considered, [1] streams holding something back
    const uint32_t *pat_cplen;      // code points: each pattern's length in code points
    uint32_t halo;                  // max_pattern_len - 1
    int mode, longest, codepoints;
};

// stream i's sequence (overlapping: only the seam's records that end past the tail are new); -> its length
__device__ __forceinline__ unsigned long long stream_view(const StreamArgs &A, int64_t i, StreamView &v) {
    const int64_t *c = A.carry + kCarryWords * i;
    const long long t = c[kCarryTail], head = min((long long)(A.B.offsets[i + 1] - A.B.offsets[i]), (long long)A.halo);
    const unsigned long long s0 = A.seam_mo[i], s1 = A.seam_mo[i + 1], c0 = A.chunk_mo[i], c1 = A.chunk_mo[i + 1];
    const unsigned long long cf = first_end_after(A.chunk_list, c0, c1, (uint32_t)head);
    const unsigned long long sf = A.mode == kModeOverlap ? first_end_after(A.seam_list, s0, s1, (uint32_t)t) : s0;
    v.chunk_base = c[kCarryFed];
    v.seam_base = c[kCarryFed] - t;
    v.chunk = A.chunk_list + cf;
    v.seam = A.seam_list + sf;
    v.ns = s1 - sf;
    return v.ns + (c1 - cf);
}

// One thread per stream: the release of this feed.  Overlapping: every record of the sequence (the emit kernel reads
// them from the lists).  Non-overlapping: the reference's selection (next_selected, as acb_count_rows follows it),
// continued from the carried restart point, up to the first pick that the release rule does not yet allow: Standard
// releases every pick (it ends in the data seen), the leftmost kinds a pick that starts at least max_pattern_len bytes
// before the end of the data seen (no later record can start before it).  Rows go to staged[], their count to
// row_offsets[i + 1].
template <int MODE>
__global__ void stream_select_kernel(StreamArgs A) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.B.n_haystacks; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t *c = A.carry + kCarryWords * i;
        const long long fed = c[kCarryFed], len = A.B.offsets[i + 1] - A.B.offsets[i];
        const long long fed_after = fed + len;
        const bool last = A.last && A.last[i];
        StreamView v;
        const unsigned long long n = stream_view(A, i, v);
        long long *out = A.staged + 4 * (A.seam_mo[i] + A.chunk_mo[i]);
        unsigned long long w = 0;
        bool pending = false;
        auto put = [&](const SelRec &m) {
            out[4 * w] = i, out[4 * w + 1] = m.pid, out[4 * w + 2] = m.start, out[4 * w + 3] = m.end;
            w++;
        };
        long long s = c[kCarryRestart];
        if (MODE == kModeOverlap) {
            w = n;
        } else {
            for (;;) {
                const unsigned long long j = next_selected<MODE>(&v, n, s, (long long)A.halo + 1, A.longest);
                if (j >= n) break;
                const SelRec m = sel_rec(&v, j);
                if (MODE == kModeLeftmost && !last && m.start + (long long)A.halo + 1 > fed_after) {
                    pending = true;
                    break;
                }
                put(m);
                s = m.end;
            }
            c[kCarryRestart] = s;
        }
        A.row_offsets[i + 1] = (int64_t)w;
        const long long t_after = min(fed_after, (long long)A.halo);
        if (A.codepoints) {
            const long long x = max(len - t_after, 0ll);
            A.cont_rows[3 * i] = 0, A.cont_rows[3 * i + 1] = x, A.cont_rows[3 * i + 2] = x;
        }
        atomicAdd(A.stats, n);
        if (!last && (pending || (MODE != kModeOverlap && s > fed_after - t_after))) atomicAdd(A.stats + 1, 1ull);
    }
}

// released row k of stream i: overlapping rows are read from the lists directly, the others from the staging area
__device__ __forceinline__ SelRec stream_row(const StreamArgs &A, int64_t i, const StreamView &v, long long k) {
    if (A.mode == kModeOverlap) return sel_rec(&v, (unsigned long long)k);
    const long long *src = A.staged + 4 * (A.seam_mo[i] + A.chunk_mo[i]);
    return {src[4 * k + 1], src[4 * k + 2], src[4 * k + 3]};
}

// Byte offsets: every released row packed at its place in rows[], grid-stride over all rows (a stream with millions of
// rows is spread over the whole grid); the stream of row g is found by a binary search in row_offsets.  Runs before
// stream_emit_kernel, which updates the carry these rows are placed with.
__global__ void stream_rows_kernel(StreamArgs A) {
    const int64_t n = A.B.n_haystacks, total = A.row_offsets[n];
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t i = 0, hi = n - 1;  // the last stream whose rows start at or before g: its rows hold g
        while (i < hi) {
            const int64_t mid = (i + hi + 1) >> 1;
            if (A.row_offsets[mid] <= g)
                i = mid;
            else
                hi = mid - 1;
        }
        StreamView v;
        if (A.mode == kModeOverlap) stream_view(A, i, v);
        const SelRec m = stream_row(A, i, v, g - A.row_offsets[i]);
        long long *dst = A.rows + 4 * g;
        dst[0] = i, dst[1] = m.pid, dst[2] = m.start, dst[3] = m.end;
    }
}

// One warp per stream: code points only, the rows packed at row_offsets[i] with positions lowered by the continuation
// bytes before them, counted from the tail on; then, for every stream, the carry: the new tail, the data fed and the
// continuation bytes before the new tail; zero for a stream that ends with this feed.
__global__ void stream_emit_kernel(StreamArgs A) {
    const uint32_t lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < A.B.n_haystacks; i += warps) {
        int64_t *c = A.carry + kCarryWords * i;
        const long long fed = c[kCarryFed], t = c[kCarryTail], cont = c[kCarryCont];
        const long long len = A.B.offsets[i + 1] - A.B.offsets[i];
        const uint8_t *seam = A.seam + A.seam_offsets[i], *chunk = A.B.bytes + A.B.offsets[i];
        // byte k of tail || chunk
        auto byte_at = [&](long long k) -> uint32_t { return k < t ? seam[k] : chunk[k - t]; };
        auto count_cont = [&](long long a, long long b) -> long long {  // continuation bytes of tail || chunk in [a, b)
            unsigned long long m = 0;
            for (long long k = a + lane; k < b; k += 32) m += is_cont_byte(byte_at(k));
            for (int d = 16; d >= 1; d >>= 1) m += __shfl_xor_sync(0xffffffffu, m, d);
            return (long long)m;
        };
        if (A.codepoints) {
            StreamView v;
            if (A.mode == kModeOverlap) stream_view(A, i, v);
            long long *dst = A.rows + 4 * A.row_offsets[i];
            const long long k_rows = A.row_offsets[i + 1] - A.row_offsets[i];
            const long long tail_start = fed - t;
            // rows are in order of end: the count runs forward once
            long long at = 0, seen = cont;
            for (long long k = 0; k < k_rows; k++) {
                const SelRec m = stream_row(A, i, v, k);
                const long long end = m.end - tail_start;
                seen += count_cont(at, end);
                at = end;
                if (lane == 0) {
                    const long long end_cp = tail_start + end - seen;
                    dst[4 * k] = i, dst[4 * k + 1] = m.pid, dst[4 * k + 2] = end_cp - (long long)A.pat_cplen[m.pid], dst[4 * k + 3] = end_cp;
                }
            }
        }
        const bool last = A.last && A.last[i];
        const long long fed_after = fed + len, t_after = last ? 0 : min(fed_after, (long long)A.halo);
        // the new tail: the last t_after bytes of tail || chunk (read from the seam and the chunk, never the old tail)
        const long long from = t + len - t_after;
        uint8_t *tail = A.tail + (uint64_t)i * A.halo;
        for (long long k = lane; k < t_after; k += 32) tail[k] = (uint8_t)byte_at(from + k);
        long long cont_after = 0;
        if (A.codepoints && !last) {
            const long long x = A.cont_rows[3 * i + 1];  // chunk bytes before the new tail: counted on the whole grid
            cont_after = cont + count_cont(0, min(from, t)) + (x - A.cont_cp[3 * i + 1]);
        }
        __syncwarp();
        if (lane == 0) {
            c[kCarryFed] = last ? 0 : fed_after;
            c[kCarryTail] = t_after;
            c[kCarryCont] = cont_after;
            if (last) c[kCarryRestart] = 0;
        }
    }
}

// ---------------------------------------------------------------------------
// Stream queries (acb_stream_advance, acb_stream_first_resolve, acb_stream_count): is_match, find_first and
// count_matches per stream, without the rows.  They use the seams and the carry of the stream search; the advance is
// the carry half of stream_emit_kernel, for feeds that make no selection (or count it without rows).
// ---------------------------------------------------------------------------

// code points: cont_rows[i] = (0, x, x), x = chunk bytes before the new tail, as stream_select_kernel writes it
__global__ void stream_cont_rows_kernel(StreamArgs A) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.B.n_haystacks; i += (int64_t)gridDim.x * blockDim.x) {
        const long long len = A.B.offsets[i + 1] - A.B.offsets[i];
        const long long x = max(len - min(A.carry[kCarryWords * i + kCarryFed] + len, (long long)A.halo), 0ll);
        A.cont_rows[3 * i] = 0, A.cont_rows[3 * i + 1] = x, A.cont_rows[3 * i + 2] = x;
    }
}

// One warp per stream: the new tail, the data fed, and (code points) the continuation bytes before the new tail; the
// whole carry is zeroed for a stream that ends with this feed.
__global__ void stream_advance_kernel(StreamArgs A) {
    const uint32_t lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < A.B.n_haystacks; i += warps) {
        int64_t *c = A.carry + kCarryWords * i;
        const long long fed = c[kCarryFed], t = c[kCarryTail], cont = c[kCarryCont];
        const long long len = A.B.offsets[i + 1] - A.B.offsets[i];
        const uint8_t *seam = A.seam + A.seam_offsets[i], *chunk = A.B.bytes + A.B.offsets[i];
        const bool last = A.last && A.last[i];
        const long long fed_after = fed + len, t_after = last ? 0 : min(fed_after, (long long)A.halo);
        const long long from = t + len - t_after;  // the new tail: bytes [from, t + len) of tail || chunk
        uint8_t *tail = A.tail + (uint64_t)i * A.halo;
        for (long long k = lane; k < t_after; k += 32) tail[k] = k + from < t ? seam[k + from] : chunk[k + from - t];
        long long cont_after = 0;
        if (A.codepoints && !last) {
            unsigned long long m = 0;  // continuation bytes of the old tail before `from`
            for (long long k = lane; k < min(from, t); k += 32) m += is_cont_byte(seam[k]);
            for (int d = 16; d >= 1; d >>= 1) m += __shfl_xor_sync(0xffffffffu, m, d);
            cont_after = cont + (long long)m + (A.cont_rows[3 * i + 1] - A.cont_cp[3 * i + 1]);
        }
        __syncwarp();
        if (lane == 0) {
            c[kCarryFed] = last ? 0 : fed_after;
            c[kCarryTail] = t_after;
            c[kCarryCont] = cont_after;
            if (last) c[kCarryRestart] = 0;
        }
    }
}

// find_first: the best candidate a stream carries, int64[n][kBestWords]: state, then (pattern, start, end) in bytes
// (absolute) and start, end in code points (a copy of the bytes' without code points)
enum : int { kBestState = 0, kBestPid = 1, kBestStart = 2, kBestEnd = 3, kBestCpStart = 4, kBestCpEnd = 5, kBestWords = 6 };
enum : int { kFirstNone = 0, kFirstPending = 1, kFirstFinal = 2 };

struct FirstArgs {
    Batch B;                          // the chunks
    const int64_t *carry;             // before this feed's advance
    const uint8_t *last;
    const uint8_t *seam;
    const int64_t *seam_offsets;
    unsigned long long *seam_keys, *chunk_keys;  // [n] each
    const long long *seam_rows, *chunk_rows;     // [n][3] decoded, bytes relative to the seam / the chunk
    const long long *seam_cp, *chunk_cp;         // [n][3] the same in code points (codepoints only)
    long long *best;                  // [n][kBestWords]
    long long *rows;                  // [n][3] the answers after this feed
    unsigned long long *stats;        // [1] streams with a pending candidate
    uint32_t max_len;
    int kind, codepoints;
};

// the streams whose keys were pre-set to 0 (their scans were skipped): the keys go back to ~0, so the rows decode none
__global__ void stream_first_unmask_kernel(FirstArgs A) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.B.n_haystacks; i += (int64_t)gridDim.x * blockDim.x) {
        const long long state = A.best[kBestWords * i + kBestState];
        if (state == kFirstFinal) A.seam_keys[i] = ~0ull;
        if (state == kFirstFinal || (state == kFirstPending && A.kind != ACB_STANDARD)) A.chunk_keys[i] = ~0ull;
    }
}

// a better than b in the order of the kind's first match (the key order of acb_find_first, on absolute positions)
__device__ __forceinline__ bool first_better(const long long *a, const long long *b, int kind) {
    if (kind == ACB_STANDARD) {
        if (a[2] != b[2]) return a[2] < b[2];  // earliest end,
        if (a[1] != b[1]) return a[1] < b[1];  // then the longest,
        return a[0] < b[0];                    // then the lowest pattern
    }
    if (a[1] != b[1]) return a[1] < b[1];  // leftmost start
    if (kind == ACB_LEFTMOST_LONGEST && a[2] != b[2]) return a[2] > b[2];
    return a[0] < b[0];
}

// One thread per stream: the carried best, the seam's candidate and the chunk's, in absolute positions; the best of
// them is final once no later data can change it (Standard: at once; leftmost: start + max_pattern_len <= F; every
// candidate on `last`).  Writes the answer row, the state, and the keys of the next feed: 0 where that scan can be
// skipped (a final answer: both; a pending leftmost candidate: the chunk's, whose records all start after it).
__global__ void stream_first_resolve_kernel(FirstArgs A) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.B.n_haystacks; i += (int64_t)gridDim.x * blockDim.x) {
        long long *b = A.best + kBestWords * i;
        const int64_t *c = A.carry + kCarryWords * i;
        const long long fed = c[kCarryFed], t = c[kCarryTail], cont = c[kCarryCont];
        const long long fed_after = fed + (A.B.offsets[i + 1] - A.B.offsets[i]);
        const bool last = A.last && A.last[i];
        long long state = b[kBestState];
        long long cur[5] = {b[kBestPid], b[kBestStart], b[kBestEnd], b[kBestCpStart], b[kBestCpEnd]};
        if (state != kFirstFinal) {
            bool have = state == kFirstPending;
            const long long *sr = A.seam_rows + 3 * i;
            if (sr[0] >= 0) {
                const long long base = fed - t, cp_base = fed - t - cont;
                const long long m[5] = {sr[0], base + sr[1], base + sr[2], A.codepoints ? cp_base + A.seam_cp[3 * i + 1] : base + sr[1],
                                        A.codepoints ? cp_base + A.seam_cp[3 * i + 2] : base + sr[2]};
                if (!have || first_better(m, cur, A.kind)) {
                    for (int k = 0; k < 5; k++) cur[k] = m[k];
                    have = true;
                }
            }
            const long long *cr = A.chunk_rows + 3 * i;
            if (cr[0] >= 0) {
                const long long m3[3] = {cr[0], fed + cr[1], fed + cr[2]};
                if (!have || first_better(m3, cur, A.kind)) {
                    long long cp_base = fed;
                    if (A.codepoints) {  // the continuation bytes before the chunk: before the tail, and in it
                        const uint8_t *seam = A.seam + A.seam_offsets[i];
                        long long tc = 0;
                        for (long long k = 0; k < t; k++) tc += is_cont_byte(seam[k]);
                        cp_base = fed - cont - tc;
                    }
                    cur[0] = m3[0], cur[1] = m3[1], cur[2] = m3[2];
                    cur[3] = A.codepoints ? cp_base + A.chunk_cp[3 * i + 1] : m3[1];
                    cur[4] = A.codepoints ? cp_base + A.chunk_cp[3 * i + 2] : m3[2];
                    have = true;
                }
            }
            if (have)
                state = (A.kind == ACB_STANDARD || last || cur[1] + (long long)A.max_len <= fed_after) ? kFirstFinal : kFirstPending;
        }
        const bool final_ = state == kFirstFinal;
        long long *row = A.rows + 3 * i;
        row[0] = final_ ? cur[0] : -1;
        row[1] = final_ ? cur[3] : -1;
        row[2] = final_ ? cur[4] : -1;
        if (last) state = kFirstNone;
        if (state == kFirstPending) atomicAdd(A.stats + 1, 1ull);
        b[kBestState] = state;
        b[kBestPid] = state ? cur[0] : 0;
        b[kBestStart] = state ? cur[1] : 0;
        b[kBestEnd] = state ? cur[2] : 0;
        b[kBestCpStart] = state ? cur[3] : 0;
        b[kBestCpEnd] = state ? cur[4] : 0;
        A.seam_keys[i] = state == kFirstFinal ? 0ull : ~0ull;
        A.chunk_keys[i] = (state == kFirstFinal || (state == kFirstPending && A.kind != ACB_STANDARD)) ? 0ull : ~0ull;
    }
}

// count_matches: the running count of stream i is what the rows stream would have released so far
struct CountArgs {
    StreamArgs S;                          // the lists, the carry (before this feed's advance), last, halo, mode, longest
    const unsigned long long *chunk_counts;  // overlapping: acb_count_overlapping's count of each chunk
    long long *running;                    // [n]
    long long *out;                        // [n] the counts after this feed
    unsigned long long *stats;             // [0] records, [1] streams holding a pick, [2] streams selected on the grid, [3] the longest
    long long *per;                        // [n][4] grid path: released count, new restart point, NEXT(restart), sequence length
    long long *long_list;                  // [n] the streams selected on the grid
    uint4 *pairs;                          // [R] successor pairs, double-buffered (jump_pair)
    uint32_t *mark;                        // [R] records on the selected chain
};

__device__ __forceinline__ void count_finish(const CountArgs &A, int64_t i, long long add, bool last) {
    const long long v = A.running[i] + add;
    A.out[i] = v;
    A.running[i] = last ? 0 : v;
}

// overlapping (Standard): a feed adds its chunk's count and the seam's records that cross the tail / head join
// (start < T < end): the others lie in the head (counted with the chunk) or in the tail (counted by earlier feeds)
__global__ void stream_count_overlap_kernel(CountArgs A) {
    const StreamArgs &S = A.S;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < S.B.n_haystacks; i += (int64_t)gridDim.x * blockDim.x) {
        const long long t = S.carry[kCarryWords * i + kCarryTail];
        const unsigned long long s1 = S.seam_mo[i + 1];
        long long cross = 0;
        for (unsigned long long j = first_end_after(S.seam_list, S.seam_mo[i], s1, (uint32_t)t); j < s1; j++) cross += S.seam_list[j].z < (uint32_t)t;
        atomicAdd(A.stats, s1 - S.seam_mo[i]);
        count_finish(A, i, (long long)A.chunk_counts[i] + cross, S.last && S.last[i]);
    }
}

// Non-overlapping, every kind: the selection continued from the carried restart point, counted up to the first pick the
// release rule does not allow yet.  A sequence of at most ACB_LONG_STRETCH records is counted by one thread
// (next_selected, as stream_select_kernel).  A longer one is selected by the whole grid: every record gets the successor
// NEXT(end), the chain from NEXT(restart) is marked by pointer jumping (select_stretches' rule), and the released count
// is the number of marked records with start + max_pattern_len <= F (all of them on `last`); the new restart point is
// the end of the last released one.  Cooperative launch.
template <int MODE>
__global__ void __launch_bounds__(kScanThreads) stream_count_kernel(CountArgs A) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const StreamArgs &S = A.S;
    const long long max_len = (long long)S.halo + 1;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long first_i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t i = (int64_t)first_i; i < S.B.n_haystacks; i += (int64_t)stride) {
        int64_t *c = S.carry + kCarryWords * i;
        const long long fed_after = c[kCarryFed] + (S.B.offsets[i + 1] - S.B.offsets[i]);
        const bool last = S.last && S.last[i];
        StreamView v;
        const unsigned long long n = stream_view(S, i, v);
        atomicAdd(A.stats, n);
        long long s = c[kCarryRestart];
        if (n > ACB_LONG_STRETCH) {
            long long *p = A.per + 4 * i;
            p[0] = 0, p[1] = s, p[2] = (long long)next_selected<MODE>(&v, n, s, max_len, S.longest), p[3] = (long long)n;
            A.long_list[atomicAdd(A.stats + 2, 1ull)] = i;
            atomicMax(A.stats + 3, n);
            continue;
        }
        long long k = 0;
        bool pending = false;
        for (;;) {
            const unsigned long long j = next_selected<MODE>(&v, n, s, max_len, S.longest);
            if (j >= n) break;
            const SelRec m = sel_rec(&v, j);
            if (MODE == kModeLeftmost && !last && m.start + max_len > fed_after) {
                pending = true;
                break;
            }
            k++;
            s = m.end;
        }
        c[kCarryRestart] = s;
        if (pending) atomicAdd(A.stats + 1, 1ull);
        count_finish(A, i, k, last);
    }
    grid.sync();
    const unsigned long long n_long = A.stats[2];
    if (n_long == 0) return;
    // the streams on the grid, one after another; record j of stream i sits at index seam_mo[i] + chunk_mo[i] + j
    for (unsigned long long q = 0; q < n_long; q++) {
        const int64_t i = A.long_list[q];
        StreamView v;
        const unsigned long long n = stream_view(S, i, v), base = S.seam_mo[i] + S.chunk_mo[i], head = (unsigned long long)A.per[4 * i + 2];
        for (unsigned long long j = first_i; j < n; j += stride) {
            const unsigned long long nx = next_selected<MODE>(&v, n, sel_rec(&v, j).end, max_len, S.longest);
            reinterpret_cast<uint2 *>(A.pairs + base + j)[0] = make_uint2(nx >= n ? kNoNext : (uint32_t)(base + nx), 1u);
            A.mark[base + j] = j == head ? 1u : 0u;
        }
    }
    grid.sync();
    const uint32_t rounds = ceil_log2(A.stats[3]);
    for (uint32_t r = 0; r < rounds; r++) {
        const int src = (int)(r & 1);
        for (unsigned long long q = 0; q < n_long; q++) {
            const int64_t i = A.long_list[q];
            const unsigned long long n = (unsigned long long)A.per[4 * i + 3], base = S.seam_mo[i] + S.chunk_mo[i];
            for (unsigned long long j = first_i; j < n; j += stride) {
                const uint32_t nx = src ? A.pairs[base + j].z : A.pairs[base + j].x;  // J_r(base + j)
                if (nx != kNoNext && A.mark[base + j]) A.mark[nx] = 1u;
                jump_pair(A.pairs, base + j, src);
            }
        }
        grid.sync();
    }
    for (unsigned long long q = 0; q < n_long; q++) {
        const int64_t i = A.long_list[q];
        StreamView v;
        const unsigned long long n = stream_view(S, i, v), base = S.seam_mo[i] + S.chunk_mo[i];
        const long long fed_after = S.carry[kCarryWords * i + kCarryFed] + (S.B.offsets[i + 1] - S.B.offsets[i]);
        const bool last = S.last && S.last[i];
        unsigned long long released = 0, held = 0;
        long long end = 0;  // (every end is positive)
        for (unsigned long long j = first_i; j < n; j += stride) {
            if (!A.mark[base + j]) continue;
            const SelRec m = sel_rec(&v, j);
            if (MODE == kModeStandard || last || m.start + max_len <= fed_after) {
                released++;
                end = max(end, m.end);
            } else {
                held++;
            }
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            released += __shfl_xor_sync(0xffffffffu, released, d);
            held += __shfl_xor_sync(0xffffffffu, held, d);
            end = max(end, (long long)__shfl_xor_sync(0xffffffffu, end, d));
        }
        if ((threadIdx.x & 31) == 0) {
            if (released) atomicAdd(reinterpret_cast<unsigned long long *>(A.per + 4 * i), released);
            if (released) atomicMax(A.per + 4 * i + 1, end);
            if (held) atomicOr(reinterpret_cast<unsigned long long *>(A.per + 4 * i + 3), 1ull << 62);
        }
    }
    grid.sync();
    for (unsigned long long q = first_i; q < n_long; q += stride) {
        const int64_t i = A.long_list[q];
        const long long *p = A.per + 4 * i;
        S.carry[kCarryWords * i + kCarryRestart] = p[1];
        if (p[3] & (1ll << 62)) atomicAdd(A.stats + 1, 1ull);
        count_finish(A, i, p[0], S.last && S.last[i]);
    }
}

// ---------------------------------------------------------------------------
// Match-mask streams (acb_stream_mask_rows, acb_stream_mask_emit): which positions of each stream lie inside a match,
// released once no later data can change them.  After a feed a stream has released [0, R), R = F - T (R = F on
// `last`); a match covering p < R starts at most p and ends by start + max_pattern_len <= F, so the rows stream has
// released it for every kind.  The caller keeps the stream search's carry, tail and seams, and the HELD flags: one u8
// per byte of the tail, the flags of [R, F).  A feed ORs its coverage into two bit spaces, one over the chunk buffer
// and one over the seam buffer; the emit then writes the flags of [R_old, R_new) and the held flags of [R_new, F_new).
// Both read the carry as it was before the feed.
// ---------------------------------------------------------------------------
struct MaskStreamArgs {
    const int64_t *offsets;         // [n + 1] the chunks
    int64_t n;
    const int64_t *carry;           // [n][kCarryWords] before this feed
    const int64_t *seam_offsets;    // [n + 1]
    const uint8_t *last;            // [n] or null
    uint32_t *chunk_mask, *seam_mask;  // bit q: byte q of the chunk buffer / of the seam buffer
    const uint8_t *held_in;         // [n][halo]: byte k = the flag of R_old + k, k < T_old
    uint8_t *held_out;              // [n][halo]: byte k = the flag of R_new + k, k < T_new
    uint8_t *flags;                 // the released flags, packed by stream
    int64_t *flag_offsets;          // [n + 1]
    int64_t *flag_starts;           // [n] the index of each stream's first released position (in units of stride)
    unsigned long long stride;      // 1: a flag per byte; ACB_TOKEN_BYTES: a flag per token (at its first byte)
    uint32_t halo;
    int overlapping;
};

// stream i's positions: r_old = F_old - T_old, f_new = F_old + chunk length, r_new = what this feed releases up to
__device__ __forceinline__ void mask_stream_range(const MaskStreamArgs &A, int64_t i, long long &r_old, long long &r_new, long long &f_new) {
    const int64_t *c = A.carry + kCarryWords * i;
    r_old = c[kCarryFed] - c[kCarryTail];
    f_new = c[kCarryFed] + (A.offsets[i + 1] - A.offsets[i]);
    r_new = (A.last && A.last[i]) ? f_new : f_new - min(f_new, (long long)A.halo);
}

__device__ __forceinline__ uint32_t mask_bit(const uint32_t *m, unsigned long long q) { return (m[q >> 5] >> (q & 31u)) & 1u; }

// the flag of byte p of stream i, r_old <= p < f_new: in the old tail the held flag OR the seam's bit; in the chunk
// the chunk's bit, OR (overlapping) the seam's bit when p lies in the head (a match that crosses the cut)
__device__ __forceinline__ uint32_t mask_stream_flag(const MaskStreamArgs &A, int64_t i, long long p) {
    const int64_t *c = A.carry + kCarryWords * i;
    const long long fed = c[kCarryFed], t = c[kCarryTail];
    if (p < fed) {
        const long long k = p - (fed - t);
        return A.held_in[(unsigned long long)i * A.halo + k] | mask_bit(A.seam_mask, (unsigned long long)(A.seam_offsets[i] + k));
    }
    const long long k = p - fed;
    uint32_t f = mask_bit(A.chunk_mask, (unsigned long long)(A.offsets[i] + k));
    if (A.overlapping && k < (long long)A.halo) f |= mask_bit(A.seam_mask, (unsigned long long)(A.seam_offsets[i] + t + k));
    return f;
}

// Non-overlapping: every released row (stream, pattern, start, end; absolute bytes) ORs its bytes into the bit spaces,
// the part in the old tail [F - T, F) into the seam's and the rest into the chunk's.  A row this feed releases was not
// released before, so it starts at or after F - T: it lies in tail || chunk.  Grid-stride over all rows.
__global__ void stream_mask_rows_kernel(MaskStreamArgs A, const long long *rows, const int64_t *row_offsets) {
    const int64_t total = row_offsets[A.n];
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const long long *r = rows + 4 * g;
        const int64_t i = r[0];
        const long long s = r[2], e = r[3];
        const long long fed = A.carry[kCarryWords * i + kCarryFed], t = A.carry[kCarryWords * i + kCarryTail];
        if (s < fed) or_bits(A.seam_mask, (unsigned long long)(A.seam_offsets[i] + s - (fed - t)), (uint32_t)(min(e, fed) - s));
        if (e > fed) {
            const long long c0 = max(s, fed);
            or_bits(A.chunk_mask, (unsigned long long)(A.offsets[i] + c0 - fed), (uint32_t)(e - c0));
        }
    }
}

// flag_offsets[i + 1] = the positions stream i releases (multiples of stride in [r_old, r_new)), flag_starts[i] = the
// first one's index
__global__ void stream_mask_count_kernel(MaskStreamArgs A) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
        long long r_old, r_new, f_new;
        mask_stream_range(A, i, r_old, r_new, f_new);
        const long long s = (long long)A.stride, first = (r_old + s - 1) / s, end = (r_new + s - 1) / s;
        A.flag_offsets[i + 1] = end - first;
        A.flag_starts[i] = first;
    }
}

// Every released flag, grid-stride over all of them (one stream with a 256 MiB feed is spread over the whole grid);
// the stream of flag g by a binary search in flag_offsets, as stream_rows_kernel.  Then the held flags of [r_new,
// f_new), grid-stride over n * halo.  held_in and held_out are different buffers: a chunk shorter than the tail
// shifts it.
__global__ void stream_mask_emit_kernel(MaskStreamArgs A) {
    const int64_t n = A.n, total = A.flag_offsets[n];
    const int64_t step = (int64_t)gridDim.x * blockDim.x, first_g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t g = first_g; g < total; g += step) {
        int64_t i = 0, hi = n - 1;  // the last stream whose flags start at or before g: its flags hold g
        while (i < hi) {
            const int64_t mid = (i + hi + 1) >> 1;
            if (A.flag_offsets[mid] <= g)
                i = mid;
            else
                hi = mid - 1;
        }
        const long long p = (A.flag_starts[i] + (g - A.flag_offsets[i])) * (long long)A.stride;
        A.flags[g] = (uint8_t)mask_stream_flag(A, i, p);
    }
    const int64_t held = n * (int64_t)A.halo;
    for (int64_t q = first_g; q < held; q += step) {
        const int64_t i = q / A.halo, k = q - i * A.halo;
        long long r_old, r_new, f_new;
        mask_stream_range(A, i, r_old, r_new, f_new);
        if (k < f_new - r_new) A.held_out[q] = (uint8_t)mask_stream_flag(A, i, r_new + k);
    }
}

}  // namespace acb

// ===========================================================================
// C ABI
// ===========================================================================
using namespace acb;

struct acb_automaton {
    Automaton *impl;
};

// Per-thread state only: the last error, the tuning knobs and the optional kernel timing belong to the calling
// thread (two automata scanned from two threads do not see each other's settings); the launch counter is atomic.
static thread_local std::string g_err;
static std::atomic<unsigned long long> g_launches{0};
static thread_local acb_tuning g_tuning = {0, 0, 0, 0, 0};  // kernel, hot_rows, segment_bytes, table, sieve_ring

// optional device timing of the dominant (scan) kernel, for bench.py's roofline
static thread_local bool g_timing = false;
static thread_local std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_timing_events;

static int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}

#define CUDA_OK(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (expr);                                                                        \
        if (e_ != cudaSuccess) return fail(ACB_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
    } while (0)

extern "C" {

const char *acb_last_error(void) { return g_err.c_str(); }
const char *acb_version(void) { return "acb200 0.2 (sm_90a)"; }
uint64_t acb_launch_count(void) { return g_launches.load(); }

int acb_timing_enable(int on) {
    g_timing = on != 0;
    return ACB_OK;
}

int acb_timing_read(double *total_ms, uint64_t *n_scans) {
    double tot = 0;
    uint64_t n = 0;
    for (auto &p : g_timing_events) {
        float ms = 0;
        CUDA_OK(cudaEventSynchronize(p.second));
        CUDA_OK(cudaEventElapsedTime(&ms, p.first, p.second));
        tot += ms;
        n++;
        cudaEventDestroy(p.first);
        cudaEventDestroy(p.second);
    }
    g_timing_events.clear();
    if (total_ms) *total_ms = tot;
    if (n_scans) *n_scans = n;
    return ACB_OK;
}

int acb_set_tuning(const acb_tuning *t) {
    if (!t) return fail(ACB_EINVAL, "null tuning");
    g_tuning = *t;
    return ACB_OK;
}

int acb_build(const uint8_t *blob, const uint64_t *offsets, uint64_t n, int match_kind, int implementation,
              acb_automaton **out) {
    if (!out || !offsets || (!blob && n && offsets[n] != 0)) return fail(ACB_EINVAL, "null argument");
    if (implementation < -1 || implementation > 2) return fail(ACB_EINVAL, "unknown implementation");
    try {
        Automaton *impl = build_automaton(blob, offsets, n, match_kind, implementation);
        *out = new acb_automaton{impl};
        return ACB_OK;
    } catch (const std::exception &e) {
        return fail(ACB_EBUILD, e.what());
    }
}

void acb_free(acb_automaton *a) {
    if (!a) return;
    delete a->impl;
    delete a;
}

uint64_t acb_num_patterns(const acb_automaton *a) { return a->impl->hdr.n_patterns; }
uint64_t acb_num_states(const acb_automaton *a) { return a->impl->hdr.n_states; }
uint32_t acb_num_columns(const acb_automaton *a) { return a->impl->hdr.n_cols; }
uint32_t acb_max_pattern_len(const acb_automaton *a) { return a->impl->hdr.max_pat_len; }
uint32_t acb_min_pattern_len(const acb_automaton *a) { return a->impl->hdr.min_pat_len; }
int acb_match_kind(const acb_automaton *a) { return (int)a->impl->hdr.match_kind; }
uint64_t acb_image_bytes(const acb_automaton *a) { return a->impl->hdr.total_bytes; }

int acb_image_write(const acb_automaton *a, void *host_dst, uint64_t dst_bytes) {
    if (!a || !host_dst) return fail(ACB_EINVAL, "null argument");
    if (dst_bytes < a->impl->hdr.total_bytes) return fail(ACB_ECAPACITY, "image buffer too small");
    std::memcpy(host_dst, a->impl->image.data(), a->impl->hdr.total_bytes);
    return ACB_OK;
}

uint64_t acb_hot_bytes(const acb_automaton *a, uint32_t max_rows) { return hot_image_bytes(*a->impl, max_rows); }

int acb_hot_build(const acb_automaton *a, const uint32_t *host_visits, uint32_t max_rows, void *host_dst, uint64_t dst_bytes) {
    if (!a || !host_dst) return fail(ACB_EINVAL, "null argument");
    if (dst_bytes < hot_image_bytes(*a->impl, max_rows)) return fail(ACB_ECAPACITY, "hot image buffer too small");
    build_hot_image(*a->impl, host_visits, max_rows, static_cast<uint8_t *>(host_dst));
    return ACB_OK;
}

uint32_t acb_hot_rows(const void *host_hot) {
    const HotHeader *h = static_cast<const HotHeader *>(host_hot);
    return (h && h->magic == kHotMagic) ? h->n_rows : 0;
}

int acb_hot_describe(const void *host_hot, acb_hot_desc *desc) {
    const HotHeader *h = static_cast<const HotHeader *>(host_hot);
    if (!h || !desc || h->magic != kHotMagic) return fail(ACB_EINVAL, "not a hot image");
    desc->rows = h->n_rows;
    desc->rows128 = h->n_rows128;
    desc->visited = h->n_visited;
    desc->reserved = 0;
    return ACB_OK;
}

uint64_t acb_sieve_build(acb_automaton *a, uint32_t bloom_bytes_max, uint32_t w_max) {
    if (!a) {
        fail(ACB_EINVAL, "null argument");
        return 0;
    }
    Automaton &A = *a->impl;
    std::lock_guard<std::mutex> lock(A.sieve_mutex);
    if (A.sieve.empty() || A.sieve_bloom_max != bloom_bytes_max || A.sieve_w_max != w_max) {
        try {
            sieve_image_build(A.pat_blob.data(), A.pat_offs.data(), A.hdr.n_patterns, bloom_bytes_max, w_max, A.sieve);
            A.sieve_bloom_max = bloom_bytes_max;
            A.sieve_w_max = w_max;
        } catch (const std::exception &e) {
            A.sieve.clear();
            fail(ACB_EBUILD, e.what());
            return 0;
        }
    }
    return A.sieve.size();
}

int acb_sieve_write(acb_automaton *a, void *host_dst, uint64_t dst_bytes) {
    if (!a || !host_dst) return fail(ACB_EINVAL, "null argument");
    Automaton &A = *a->impl;
    std::lock_guard<std::mutex> lock(A.sieve_mutex);
    if (A.sieve.empty()) return fail(ACB_EINVAL, "acb_sieve_build has not been called");
    if (dst_bytes < A.sieve.size()) return fail(ACB_ECAPACITY, "sieve image buffer too small");
    std::memcpy(host_dst, A.sieve.data(), A.sieve.size());
    return ACB_OK;
}

int acb_sieve_describe(const void *host_sieve, acb_sieve_desc *d) {
    const SieveHeader *h = static_cast<const SieveHeader *>(host_sieve);
    if (!h || !d || h->magic != kSieveMagic) return fail(ACB_EINVAL, "not a sieve image");
    d->window = h->W;
    d->last_level = h->last_level;
    d->probes = h->n_probes;
    d->bloom_bytes = h->bloom_words * 4;
    d->nodes = h->n_nodes;
    d->keys = h->n_keys;
    d->filter_entries = h->n_filter_entries;
    d->table_slots = h->ht_mask + 1;
    return ACB_OK;
}

// tasks of the sieve kernel: a multiple of 512 bytes (tuning.segment_bytes when the sieve kernel is forced, else 16 KiB)
static uint32_t sieve_task_bytes() {
    uint32_t t = (g_tuning.kernel == 5 && g_tuning.segment_bytes > 0) ? (uint32_t)g_tuning.segment_bytes : 16384u;
    t = (t + 511u) & ~511u;
    return t < 512u ? 512u : t;
}

int acb_plan_scan(const acb_automaton *a, const void *dev_bytes, uint64_t total_bytes, uint64_t n_haystacks, acb_plan *plan) {
    if (!a || !plan) return fail(ACB_EINVAL, "null argument");
    const uint32_t L = a->impl->hdr.max_pat_len;
    // the warm-up must cover a whole longest pattern so that the guessed state equals the true one
    // whenever the true scanner did not restart inside it
    uint32_t warm = (L + 15u) & ~15u;
    if (warm < 16) warm = 16;
    uint32_t seg = g_tuning.segment_bytes > 0 ? (uint32_t)g_tuning.segment_bytes : 1024u;
    if (seg < 8 * warm) seg = 8 * warm;
    seg = (seg + 63u) & ~63u;
    const uint64_t mis = reinterpret_cast<uintptr_t>(dev_bytes) & 63u;  // segment 0 starts at the 64-byte aligned address before the buffer
    plan->segment_bytes = seg;
    plan->warm_bytes = warm;
    plan->n_segments = (total_bytes + mis + seg - 1) / seg;
    uint64_t stride = 1;
    if (n_haystacks > 1) {
        const uint64_t avg = total_bytes / n_haystacks;
        stride = (avg + seg / 2) / seg;
        if (stride < 1) stride = 1;
        if (stride > 65536) stride = 65536;
    }
    plan->lane_stride = (uint32_t)stride;
    // the sieve kernel's tasks: a grid anchored at the 512-byte aligned address at or before the buffer
    plan->task_bytes = sieve_task_bytes();
    const uint64_t mis512 = reinterpret_cast<uintptr_t>(dev_bytes) & 511u;
    const uint64_t n_tasks = (total_bytes + mis512 + plan->task_bytes - 1) / plan->task_bytes;
    const uint64_t seg_units = 2 * plan->n_segments;
    plan->n_units = seg_units > n_haystacks ? seg_units : n_haystacks;
    if (plan->n_units < n_tasks) plan->n_units = n_tasks;
    if (plan->n_units < 1) plan->n_units = 1;
    const uint64_t tiles = (plan->n_units + kScanTile - 1) / kScanTile;
    const uint64_t per_piece = plan->n_segments > n_tasks ? plan->n_segments : n_tasks;  // segments or tasks, whichever kernel runs
    // [0..7] counters (kAcc* in capi.cu) | unit tile sums | cont tile sums | cont_cum (pieces + 1) | sieve cont tails (u32)
    // | table walkers' epilogue: one "has matches" bit per unit
    plan->scratch_words = 8 + (tiles + 1) + (tiles + 1) + (per_piece + 2) + (per_piece / 2 + 2) + (plan->n_units / 64 + 2);
    return ACB_OK;
}

// as many windows of text per warp as fit next to the filters (a power of two): the more, the fuller the rounds of the
// later stages when survivors are rare.  tuning.sieve_ring caps it (rounded down to a power of two); 0 = nothing fits
uint32_t acb_sieve_ring(uint32_t bloom_bytes, uint32_t smem_optin) {
    auto fits = [&](uint32_t ring) { return uint64_t(bloom_bytes) + sieve_smem_bytes(0, ring, false) <= smem_optin; };  // (no wrap)
    uint32_t ring = kRingMax;
    if (g_tuning.sieve_ring > 0)
        while (ring > (uint32_t)g_tuning.sieve_ring) ring >>= 1;
    while (ring > 1 && !fits(ring)) ring >>= 1;
    return fits(ring) ? ring : 0u;
}

}  // extern "C"

namespace {

struct DeviceInfo {
    int device = -1;
    int sms = 0;
    int max_smem_optin = 0;
};

int device_info(DeviceInfo &d) {
    static thread_local DeviceInfo cache;
    int dev;
    CUDA_OK(cudaGetDevice(&dev));
    if (cache.device != dev) {
        cache.device = dev;
        CUDA_OK(cudaDeviceGetAttribute(&cache.sms, cudaDevAttrMultiProcessorCount, dev));
        CUDA_OK(cudaDeviceGetAttribute(&cache.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    }
    d = cache;
    return ACB_OK;
}

DevImage make_view(const ImageHeader &h, const void *dev_image) {
    const uint8_t *b = static_cast<const uint8_t *>(dev_image);
    DevImage im;
    im.colmap = b + h.off_colmap;
    im.trans = reinterpret_cast<const uint32_t *>(b + h.off_trans);
    im.match_off = reinterpret_cast<const uint32_t *>(b + h.off_match_off);
    im.match_pid = reinterpret_cast<const uint32_t *>(b + h.off_match_pid);
    im.pat_len = reinterpret_cast<const uint32_t *>(b + h.off_pat_len);
    im.pat_cplen = reinterpret_cast<const uint32_t *>(b + h.off_pat_cplen);
    im.n_cols = h.n_cols;
    im.col_lo = h.col_lo;
    im.n_states = h.n_states;
    im.col_mode = h.col_mode;
    return im;
}

// dev_hot points at a device copy of a hot image; hot_rows is its row count (the
// host knows it: acb_hot_rows on the host copy), because the header lives on the device
int make_hot_view(const acb_automaton *a, const void *dev_hot, const acb_hot_desc &desc, DevHot &v) {
    const ImageHeader &ih = a->impl->hdr;
    const uint32_t hot_rows = desc.rows;
    if (hot_rows < 1 || (uint64_t)hot_rows * ih.n_cols * 2 > 65535 || desc.rows128 > 255)
        return fail(ACB_EINVAL, "bad hot image description");
    auto align16 = [](uint64_t x) { return (x + 15) & ~uint64_t(15); };
    const uint8_t *b = static_cast<const uint8_t *>(dev_hot);
    uint64_t off = align16(sizeof(HotHeader));
    v.table = reinterpret_cast<const uint16_t *>(b + off);
    off = align16(off + uint64_t(hot_rows + 1) * ih.n_cols * 2);
    v.hot2full = reinterpret_cast<const uint32_t *>(b + off);
    off = align16(off + uint64_t(hot_rows + 1) * 4);
    v.full2hot = reinterpret_cast<const uint16_t *>(b + off);
    v.n_rows = hot_rows;
    off = align16(off + uint64_t(ih.n_states) * 2);
    v.table128 = reinterpret_cast<const uint16_t *>(b + off);
    v.n_rows128 = desc.rows128;
    return ACB_OK;
}

template <int MODE, bool CP>
int launch_plain(const DevImage &im, const Batch &B, const Sink &out, const DeviceInfo &d, cudaStream_t st) {
    const int threads = 128;
    int64_t blocks = (B.n_haystacks + threads - 1) / threads;
    const int64_t cap = (int64_t)d.sms * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    scan_plain_kernel<MODE, CP><<<(unsigned)blocks, threads, 0, st>>>(im, B, out);
    g_launches++;
    return ACB_OK;
}

template <int MODE, bool CP, int COLMODE, int V>
int launch_staged(const DevImage &im, const DevHot &hot, const Batch &B, const SegPlan &P, const Sink &out, const SegOut &seg_out,
                  const DeviceInfo &d, unsigned int *task_counter, unsigned long long *trap_stats, cudaStream_t st) {
    auto kern = scan_staged_kernel<MODE, CP, COLMODE, V>;
    constexpr int kWarpsMax = V == 1 ? kMaxWarps : kMaxWarps2;
    const uint64_t q = P.lane_stride;
    const uint64_t tasks = ((uint64_t)P.n_segments + 32 * V * q - 1) / (32 * V * q) * q;
    const int ctas = d.sms;
    int warps = (int)((tasks + ctas - 1) / ctas);
    if (warps < 4) warps = 4;
    // as many warps as fit: the scan is a chain of dependent shared-memory loads per lane, more warps hide more of
    // it; balancing the last round of tasks instead was not better
    if (warps > kWarpsMax) warps = kWarpsMax;
    const uint32_t row_bytes = COLMODE == kColAscii ? kAsciiCols * 2 : im.n_cols * 2;
    const uint32_t stage_bytes = (uint32_t)warps * V * (2 * kStageBytes + kMetaBytes);
    const uint32_t budget = (uint32_t)d.max_smem_optin;
    if (budget < stage_bytes + kStageOffset + 3 * (row_bytes + 4) + 256) return fail(ACB_ECUDA, "not enough shared memory for the staged kernel");
    uint32_t rows = (budget - stage_bytes - kStageOffset - 256) / (row_bytes + 4);  // includes the trap row; +4: the row's hot2full entry
    // table entries are 16-bit shared-memory ADDRESSES: the table (it starts dynamic shared memory) must end below 64 KB
    if (rows > (60u * 1024u) / row_bytes) rows = (60u * 1024u) / row_bytes;
    if (COLMODE == kColAscii) rows -= 1;                                        // ... and the guard row behind it
    uint32_t H = rows - 1;
    const uint32_t have = COLMODE == kColAscii ? hot.n_rows128 : hot.n_rows;
    if (H > have) H = have;
    if (g_tuning.hot_rows > 0 && (uint32_t)g_tuning.hot_rows < H) H = (uint32_t)g_tuning.hot_rows;
    if (H < 1) return fail(ACB_ECUDA, "rows too wide for the staged kernel");
    const uint32_t hot_bytes = (((H + 1 + (COLMODE == kColAscii ? 1 : 0)) * row_bytes) + 127u) & ~127u;
    const uint32_t smem = hot_bytes + kStageOffset + (((H + 1) * 4 + 127u) & ~127u) + stage_bytes;
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)budget));
    kern<<<ctas, warps * 32, smem, st>>>(im, hot, B, P, out, seg_out, H, hot_bytes, task_counter, trap_stats);
    g_launches++;
    return ACB_OK;
}

// how many 128-wide rows fit next to the staging buffers of a full CTA
uint32_t ascii_rows_that_fit(const DeviceInfo &d) {
    const uint32_t stage_bytes = (uint32_t)kMaxWarps * (2 * kStageBytes + kMetaBytes);
    const uint32_t budget = (uint32_t)d.max_smem_optin;
    if (budget < stage_bytes + kStageOffset + 128 + 2 * kAsciiCols * 2) return 0;
    uint32_t rows = (budget - stage_bytes - kStageOffset - 256) / (kAsciiCols * 2 + 4);
    if (rows > (60u * 1024u) / (kAsciiCols * 2)) rows = (60u * 1024u) / (kAsciiCols * 2);  // 16-bit row addresses
    return rows - 2;  // minus the trap row and the guard row
}

template <int MODE, bool CP>
int launch_staged_cols(const ImageHeader &h, const DevImage &im, const DevHot &hot, const Batch &B, const SegPlan &P, const Sink &out,
                       const SegOut &seg_out, const DeviceInfo &d, unsigned int *task_counter, unsigned long long *trap_stats,
                       cudaStream_t st, bool ascii, int per_lane) {
#define ACB_GO(COLS)                                                                                                        \
    (per_lane == 2 ? launch_staged<MODE, CP, COLS, 2>(im, hot, B, P, out, seg_out, d, task_counter, trap_stats, st)      \
                   : launch_staged<MODE, CP, COLS, 1>(im, hot, B, P, out, seg_out, d, task_counter, trap_stats, st))
    if (ascii) return ACB_GO(kColAscii);
    if (h.col_mode == kColRange) return ACB_GO(kColRange);
    return ACB_GO(kColClass);
#undef ACB_GO
}

template <int MODE, bool CP>
int launch_global(const DevImage &im, const Batch &B, const SegPlan &P, const Sink &out, const SegOut &seg_out, const DeviceInfo &d,
                  cudaStream_t st) {
    int64_t blocks = (P.n_segments + 255) / 256;
    const int64_t cap = (int64_t)d.sms * 64;  // grid-stride beyond that
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    scan_global_kernel<MODE, CP><<<(unsigned)blocks, 256, 0, st>>>(im, B, P, out, seg_out);
    g_launches++;
    return ACB_OK;
}

inline int epilogue_blocks_per_sm(int max_bps, uint64_t n_units) {
    static const int forced = [] {
        const char *e = std::getenv("ACB200_EPILOGUE_BPS");
        return e ? std::atoi(e) : 0;
    }();
    (void)n_units;
    int b = forced > 0 ? forced : max_bps;  // (more blocks per SM beat one: the phases are short and latency bound)
    return b > max_bps ? max_bps : (b < 1 ? 1 : b);
}

template <int MODE, bool CP>
int launch_epilogue(EpilogueArgs &E, const DeviceInfo &d, cudaStream_t st) {
    auto kern = epilogue_kernel<MODE, CP>;
    static thread_local int blocks_per_sm[3][2] = {{0, 0}, {0, 0}, {0, 0}};
    static thread_local int cached_device = -1;  // the occupancy answer belongs to a device
    if (cached_device != d.device) {
        for (auto &row : blocks_per_sm) row[0] = row[1] = 0;
        cached_device = d.device;
    }
    int &bps = blocks_per_sm[MODE][CP ? 1 : 0];
    if (bps == 0) {
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kern, kScanThreads, 0));
        if (bps < 1) return fail(ACB_ECUDA, "epilogue kernel does not fit on an SM");
        if (bps > 4) bps = 4;
    }
    void *args[] = {&E};
    const int use_bps = epilogue_blocks_per_sm(bps, E.n_items);
    CUDA_OK(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(kern), dim3(d.sms * use_bps), dim3(kScanThreads), args, 0, st));
    g_launches++;
    return ACB_OK;
}


DevSieve make_sieve_view(const SieveHeader &h, const void *dev_sieve) {
    const uint8_t *b = static_cast<const uint8_t *>(dev_sieve);
    DevSieve v;
    v.bloom = reinterpret_cast<const uint32_t *>(b + h.off_bloom);
    v.ht = reinterpret_cast<const SieveSlot *>(b + h.off_ht);
    v.na = reinterpret_cast<const SieveNodeA *>(b + h.off_node_a);
    v.nb = reinterpret_cast<const SieveNodeB *>(b + h.off_node_b);
    v.pids = reinterpret_cast<const uint32_t *>(b + h.off_pids);
    v.W = h.W;
    v.last_level = h.last_level;
    v.n_probes = h.n_probes;
    v.bloom_words = h.bloom_words;
    v.prim_words = h.prim_words;
    v.ht_size = h.ht_mask + 1;
    v.max_pat_len = h.max_pat_len;
    v.term_levels = h.term_levels;
    return v;
}

// MODE kSieveAny (acb_any_match) / kSieveFirst + kind (acb_find_first): hay_cont carries the flags / keys and task_cont
// the two skip counters, out goes unused
// F: each haystack's pattern set (sieve_scan_filtered_kernel), or null
template <bool CP, int MODE = kSieveList>
int launch_sieve(const DevSieve &sv, const Batch &B, SievePlan &P, const Sink &out, uint32_t *task_cont, uint32_t *hay_cont,
                 unsigned int *task_counter, const DeviceInfo &d, cudaStream_t st, const SieveFilter *F = nullptr) {
    const uint32_t ring = acb_sieve_ring(sv.bloom_words * 4, (uint32_t)d.max_smem_optin);
    if (ring == 0) return fail(ACB_ECUDA, "the sieve's filters do not fit in shared memory (rebuild them with a smaller bloom_bytes_max)");
    const uint32_t smem = sieve_smem_bytes(sv.bloom_words * 4, ring, CP);
    P.ring = ring;
#define ACB_SIEVE_GO(WC)                                                                                      \
    do {                                                                                                      \
        if constexpr (MODE != kSievePatterns) {                                                               \
            if (F) {                                                                                          \
                auto kern = sieve_scan_filtered_kernel<CP, WC, MODE>;                                         \
                CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, d.max_smem_optin)); \
                kern<<<d.sms, kSieveThreads, smem, st>>>(sv, B, P, out, task_cont, hay_cont, task_counter, *F); \
                break;                                                                                        \
            }                                                                                                 \
        }                                                                                                     \
        auto kern = sieve_scan_kernel<CP, WC, MODE>;                                                          \
        CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, d.max_smem_optin));   \
        kern<<<d.sms, kSieveThreads, smem, st>>>(sv, B, P, out, task_cont, hay_cont, task_counter);           \
    } while (0)
    if (sv.W < 4)
        ACB_SIEVE_GO(0);
    else if (sv.W == 4)
        ACB_SIEVE_GO(1);
    else if (sv.W == 5)
        ACB_SIEVE_GO(3);
    else
        ACB_SIEVE_GO(2);
#undef ACB_SIEVE_GO
    g_launches++;
    return ACB_OK;
}

template <int MODE, bool CP>
int launch_sieve_epilogue(SieveEpiArgs &E, const DeviceInfo &d, cudaStream_t st) {
    auto kern = sieve_epilogue_kernel<MODE, CP>;
    static thread_local int blocks_per_sm[3][2] = {{0, 0}, {0, 0}, {0, 0}};
    static thread_local int cached_device = -1;
    if (cached_device != d.device) {
        for (auto &row : blocks_per_sm) row[0] = row[1] = 0;
        cached_device = d.device;
    }
    int &bps = blocks_per_sm[MODE][CP ? 1 : 0];
    if (bps == 0) {
        CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kern, kScanThreads, 0));
        if (bps < 1) return fail(ACB_ECUDA, "epilogue kernel does not fit on an SM");
        if (bps > 4) bps = 4;
    }
    void *args[] = {&E};
    const uint64_t n_work = E.n_tasks > (uint64_t)E.B.n_haystacks ? E.n_tasks : (uint64_t)E.B.n_haystacks;
    const int use_bps = epilogue_blocks_per_sm(bps, n_work);
    CUDA_OK(cudaLaunchCooperativeKernel(reinterpret_cast<void *>(kern), dim3(d.sms * use_bps), dim3(kScanThreads), args, 0, st));
    g_launches++;
    return ACB_OK;
}

// a cooperative launch of the count kernels: every block resident at once (at most 4 per SM, as the epilogues)
int launch_cooperative(const void *kern, void **args, const DeviceInfo &d, cudaStream_t st) {
    int bps = 0;
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kern, kScanThreads, 0));
    if (bps < 1) return fail(ACB_ECUDA, "count kernel does not fit on an SM");
    if (bps > 4) bps = 4;
    CUDA_OK(cudaLaunchCooperativeKernel(kern, dim3(d.sms * bps), dim3(kScanThreads), args, 0, st));
    g_launches++;
    return ACB_OK;
}

template <int MODE>
int launch_sieve_count_epilogue(SieveEpiArgs &E, unsigned long long *counts, const DeviceInfo &d, cudaStream_t st) {
    void *args[] = {&E, &counts};
    return launch_cooperative(reinterpret_cast<const void *>(sieve_count_epilogue_kernel<MODE>), args, d, st);
}

template <int MODE>
int launch_sieve_pattern_epilogue(SieveEpiArgs &E, unsigned long long *pattern_counts, const DeviceInfo &d, cudaStream_t st) {
    void *args[] = {&E, &pattern_counts};
    return launch_cooperative(reinterpret_cast<const void *>(sieve_pattern_epilogue_kernel<MODE>), args, d, st);
}

// acb_match_mask_*'s output: the u32 bitmask and the bit of the buffer's byte 0
struct MaskBits {
    uint32_t *mask;
    unsigned long long bit_base;
};

template <int MODE>
int launch_sieve_mask_epilogue(SieveEpiArgs &E, const MaskBits &mb, const DeviceInfo &d, cudaStream_t st) {
    uint32_t *mask = mb.mask;
    unsigned long long bit_base = mb.bit_base;
    void *args[] = {&E, &mask, &bit_base};
    return launch_cooperative(reinterpret_cast<const void *>(sieve_mask_epilogue_kernel<MODE>), args, d, st);
}

// acb_pattern_hits' counter rows
struct HitRows {
    uint32_t *rows;
    unsigned long long words;
    uint32_t n_patterns;
};

template <int MODE>
int launch_sieve_hits_epilogue(SieveEpiArgs &E, const HitRows &hr, const DeviceInfo &d, cudaStream_t st) {
    uint32_t *rows = hr.rows;
    unsigned long long words = hr.words;
    uint32_t n_patterns = hr.n_patterns;
    void *args[] = {&E, &rows, &words, &n_patterns};
    return launch_cooperative(reinterpret_cast<const void *>(sieve_hits_epilogue_kernel<MODE>), args, d, st);
}

int sieve_header(const acb_automaton *a, SieveHeader &sh) {
    std::lock_guard<std::mutex> lock(a->impl->sieve_mutex);
    if (a->impl->sieve.size() < sizeof(SieveHeader)) return fail(ACB_EINVAL, "acb_sieve_build has not been called");
    std::memcpy(&sh, a->impl->sieve.data(), sizeof(sh));
    return ACB_OK;
}

int unsupported_overlapping(const acb_automaton *a) {
    const int kind = (int)a->impl->hdr.match_kind;
    return fail(ACB_EUNSUPPORTED, std::string("match kind ") + (kind == ACB_LEFTMOST_FIRST ? "LeftmostFirst" : "LeftmostLongest") +
                                      " does not support overlapping searches");
}

// acb_pattern_filter -> the kernels' view; ACB_EINVAL (before any device work) for a malformed descriptor.  A null
// descriptor is no filter (*out stays unset, *use false).
int filter_view(const acb_automaton *a, const acb_pattern_filter *f, int64_t n_haystacks, SieveFilter &out, bool &use) {
    use = f != nullptr;
    if (!f) return ACB_OK;
    if (f->n_sets == 0) return fail(ACB_EINVAL, "pattern filter: n_sets must be at least 1");
    if (!f->dev_set_bits) return fail(ACB_EINVAL, "pattern filter: null dev_set_bits");
    if (f->index_bytes != 4 && f->index_bytes != 8) return fail(ACB_EINVAL, "pattern filter: index_bytes must be 4 or 8");
    if (!f->dev_set_index && n_haystacks > 0) return fail(ACB_EINVAL, "pattern filter: null dev_set_index");
    out.bits = f->dev_set_bits;
    out.index = f->dev_set_index;
    out.n_sets = f->n_sets;
    out.words = (uint32_t)((a->impl->hdr.n_patterns + 31) / 32);
    out.index_bytes = (uint32_t)f->index_bytes;
    return ACB_OK;
}

// acb_any_match (mode kSieveAny, out = u8 flags), acb_find_first (kSieveFirst + kind, out = u64 keys),
// acb_count_overlapping (kSieveCount, out = u64 counts per haystack), acb_pattern_counts_overlapping (kSievePatterns,
// out = u64 counts per pattern) and acb_match_mask_overlapping (kSieveCover, out = u32 mask words, from bit_base): one
// launch of the sieve kernel in a mode that writes no list
int sieve_early_scan(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                     int64_t n_haystacks, uint64_t total_bytes, void *dev_out, uint64_t *dev_scratch, void *stream, int mode,
                     const acb_pattern_filter *filter = nullptr, uint64_t bit_base = 0) {
    if (!a || !dev_sieve || !dev_offsets || !dev_out || !dev_scratch || (total_bytes && !dev_bytes)) return fail(ACB_EINVAL, "null argument");
    if (n_haystacks < 0 || n_haystacks > 0xfffffffell) return fail(ACB_EINVAL, "n_haystacks out of range (0 .. 2^32 - 2)");
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (scan larger inputs in windows)");
    SieveFilter F;
    bool filtered;
    if (int rc = filter_view(a, filter, n_haystacks, F, filtered)) return rc;
    if ((mode == kSieveCount || mode == kSievePatterns || mode == kSieveCover) && a->impl->hdr.match_kind != ACB_STANDARD)
        return unsupported_overlapping(a);
    SieveHeader sh;
    if (int rc = sieve_header(a, sh)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemsetAsync(dev_scratch, 0, kAnyScratchWords * sizeof(uint64_t), st));
    if (n_haystacks == 0 || total_bytes == 0) return ACB_OK;
    acb_plan plan;
    acb_plan_scan(a, dev_bytes, total_bytes, (uint64_t)n_haystacks, &plan);
    SievePlan SP;
    SP.origin = -(int64_t)(reinterpret_cast<uintptr_t>(dev_bytes) & 511u);
    SP.task_bytes = plan.task_bytes;
    SP.n_tasks = (int64_t)((total_bytes + (uint64_t)(-SP.origin) + plan.task_bytes - 1) / plan.task_bytes);
    SP.buf_bytes = total_bytes;
    SP.avg_len = total_bytes / (uint64_t)n_haystacks;
    if (SP.avg_len < 1) SP.avg_len = 1;
    const Batch B{dev_bytes, dev_offsets, n_haystacks};
    const DevSieve sv = make_sieve_view(sh, dev_sieve);
    unsigned long long *scr = reinterpret_cast<unsigned long long *>(dev_scratch);
    // (the kernel's code-point pointers carry the skip counters and the flags / keys in these modes)
    uint32_t *skipped = reinterpret_cast<uint32_t *>(scr + 1), *out = static_cast<uint32_t *>(dev_out);
    unsigned int *counter = reinterpret_cast<unsigned int *>(scr);
    int rc;
    const SieveFilter *Fp = filtered ? &F : nullptr;
    switch (mode) {
        case kSieveAny: rc = launch_sieve<false, kSieveAny>(sv, B, SP, Sink{}, skipped, out, counter, d, st, Fp); break;
        case kSieveFirst + ACB_STANDARD: rc = launch_sieve<false, kSieveFirst + ACB_STANDARD>(sv, B, SP, Sink{}, skipped, out, counter, d, st, Fp); break;
        case kSieveFirst + ACB_LEFTMOST_FIRST: rc = launch_sieve<false, kSieveFirst + ACB_LEFTMOST_FIRST>(sv, B, SP, Sink{}, skipped, out, counter, d, st, Fp); break;
        case kSieveFirst + ACB_LEFTMOST_LONGEST: rc = launch_sieve<false, kSieveFirst + ACB_LEFTMOST_LONGEST>(sv, B, SP, Sink{}, skipped, out, counter, d, st, Fp); break;
        case kSieveCount: rc = launch_sieve<false, kSieveCount>(sv, B, SP, Sink{}, skipped, out, counter, d, st, Fp); break;
        case kSievePatterns: rc = launch_sieve<false, kSievePatterns>(sv, B, SP, Sink{}, skipped, out, counter, d, st); break;
        case kSieveCover: {
            Sink cover{};
            cover.cap = bit_base;  // (the list's capacity carries the mask's first bit in this mode)
            rc = launch_sieve<false, kSieveCover>(sv, B, SP, cover, skipped, out, counter, d, st, Fp);
            break;
        }
        default: return fail(ACB_EINVAL, "unknown match kind");
    }
    if (rc) return rc;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int check_ws(const acb_workspace *ws) {
    if (!ws || !ws->dev_raw || !ws->dev_raw_seq || !ws->dev_raw_unit || !ws->dev_raw_aux || !ws->dev_unit_counts ||
        !ws->dev_unit_offsets || !ws->dev_seg_info || !ws->dev_scratch || !ws->dev_total || !ws->dev_out ||
        !ws->dev_match_offsets)
        return fail(ACB_EINVAL, "workspace has a null buffer");
    return ACB_OK;
}

// The sieve's list scan: the scan kernel, then the ordering epilogue -- acb_scan_batch's kernel 5 (counts == null:
// the list, or its selection, in dev_out), acb_count_non_overlapping (counts: the count epilogue writes them) or
// acb_pattern_counts_non_overlapping (counts, by_pattern: the pattern epilogue adds to them) or acb_pattern_hits (hits:
// the hits epilogue, mode kModeOverlap for the overlapping search) or acb_match_mask_non_overlapping (mb: the mask
// epilogue ORs the selection's bytes into the mask).  For the counts, the hits and the mask the raw records go to
// dev_raw and are ordered into dev_out, so that dev_raw is free for the pairs.
int sieve_list_scan(const acb_automaton *a, const void *dev_sieve, const Batch &B, uint64_t total_bytes, int mode, bool cp,
                    const uint32_t *pat_cplen, const acb_plan *plan, const acb_workspace *ws, const DeviceInfo &d, cudaStream_t st,
                    unsigned long long *counts, bool by_pattern = false, const HitRows *hits = nullptr, const SieveFilter *F = nullptr,
                    const MaskBits *mb = nullptr) {
    const ImageHeader &h = a->impl->hdr;
    const int kind = (int)h.match_kind;
    const uint8_t *dev_bytes = B.bytes;
    const int64_t n_haystacks = B.n_haystacks;
    int rc;
    unsigned long long *totals = reinterpret_cast<unsigned long long *>(ws->dev_total);
    unsigned int *task_counter = reinterpret_cast<unsigned int *>(ws->dev_scratch);
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(ws->dev_scratch);  // zero between scans (see kAcc*)
    unsigned long long *unit_offsets = reinterpret_cast<unsigned long long *>(ws->dev_unit_offsets);
    unsigned long long *match_offsets = reinterpret_cast<unsigned long long *>(ws->dev_match_offsets);
    Sink out;
    out.raw_seq = ws->dev_raw_seq;
    out.raw_unit = ws->dev_raw_unit;
    out.raw_aux = ws->dev_raw_aux;
    out.unit_counts = ws->dev_unit_counts;
    out.raw_total = acc + kAccRaw;
    SieveHeader sh;
    if ((rc = sieve_header(a, sh))) return rc;
    const DevSieve sv = make_sieve_view(sh, dev_sieve);
    SievePlan SP;
    SP.origin = -(int64_t)(reinterpret_cast<uintptr_t>(dev_bytes) & 511u);
    SP.task_bytes = plan->task_bytes;
    SP.n_tasks = (int64_t)((total_bytes + (uint64_t)(-SP.origin) + plan->task_bytes - 1) / plan->task_bytes);
    SP.buf_bytes = total_bytes;
    SP.avg_len = total_bytes / (uint64_t)n_haystacks;
    if (SP.avg_len < 1) SP.avg_len = 1;
    const uint64_t cap = ws->raw_capacity < ws->out_capacity ? ws->raw_capacity : ws->out_capacity;
    // scratch: counters | unit tile sums | cont tile sums | cont_cum | cont tails (u32)
    const uint64_t tiles_max = (plan->n_units + kScanTile - 1) / kScanTile;
    unsigned long long *tile_sums = acc + kAccWords;
    unsigned long long *cont_tiles = tile_sums + tiles_max + 1;
    unsigned long long *cont_cum = cont_tiles + tiles_max + 1;
    const uint64_t per_piece = plan->n_segments > (uint64_t)SP.n_tasks ? plan->n_segments : (uint64_t)SP.n_tasks;
    uint32_t *cont_tail = reinterpret_cast<uint32_t *>(cont_cum + per_piece + 2);
    // a non-overlapping search orders the list into dev_raw's place and packs its selection into dev_out, so its
    // raw records go through dev_out first (a count packs nothing: dev_raw -> dev_out)
    const bool in_raw = mode == kModeOverlap || counts || hits || mb;
    out.raw = in_raw ? ws->dev_raw : ws->dev_out;
    out.cap = cap;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (g_timing) {
        CUDA_OK(cudaEventCreate(&e0));
        CUDA_OK(cudaEventCreate(&e1));
        CUDA_OK(cudaEventRecord(e0, st));
    }
    // code points: the continuation bytes each task saw before a haystack that starts in it, per haystack; lives in
    // the match_offsets buffer until the epilogue's last phases write the offsets there
    uint32_t *hay_cont = reinterpret_cast<uint32_t *>(match_offsets);
    rc = cp ? launch_sieve<true>(sv, B, SP, out, cont_tail, hay_cont, task_counter, d, st, F)
            : launch_sieve<false>(sv, B, SP, out, cont_tail, hay_cont, task_counter, d, st, F);
    if (rc) return rc;
    CUDA_OK(cudaGetLastError());
    if (e1) {
        CUDA_OK(cudaEventRecord(e1, st));
        g_timing_events.emplace_back(e0, e1);
    }
    SieveEpiArgs E;
    E.B = B;
    E.unit_counts = ws->dev_unit_counts;
    E.n_tasks = (uint64_t)SP.n_tasks;
    E.tile_sums = tile_sums;
    E.unit_offsets = unit_offsets;
    E.cont_tail = cont_tail;
    E.hay_cont = hay_cont;
    E.cont_tiles = cont_tiles;
    E.cont_cum = cont_cum;
    E.raw = out.raw;
    E.raw_seq = ws->dev_raw_seq;
    E.raw_unit = ws->dev_raw_unit;
    E.raw_aux = ws->dev_raw_aux;
    E.raw_cap = cap;
    E.ordered = in_raw ? ws->dev_out : ws->dev_raw;
    E.final_out = ws->dev_out;
    E.out_cap = cap;
    E.pat_cplen = pat_cplen;
    E.origin = SP.origin;
    E.task_bytes = SP.task_bytes;
    E.max_pat_len = h.max_pat_len;
    E.longest = kind == ACB_LEFTMOST_LONGEST ? 1 : 0;
    E.totals = totals;
    E.acc = acc;
    E.match_offsets = match_offsets;
    if (mb)
        rc = mode == kModeStandard ? launch_sieve_mask_epilogue<kModeStandard>(E, *mb, d, st) : launch_sieve_mask_epilogue<kModeLeftmost>(E, *mb, d, st);
    else if (hits)
        rc = mode == kModeStandard   ? launch_sieve_hits_epilogue<kModeStandard>(E, *hits, d, st)
             : mode == kModeLeftmost ? launch_sieve_hits_epilogue<kModeLeftmost>(E, *hits, d, st)
                                     : launch_sieve_hits_epilogue<kModeOverlap>(E, *hits, d, st);
    else if (counts && by_pattern)
        rc = mode == kModeStandard ? launch_sieve_pattern_epilogue<kModeStandard>(E, counts, d, st) : launch_sieve_pattern_epilogue<kModeLeftmost>(E, counts, d, st);
    else if (counts)
        rc = mode == kModeStandard ? launch_sieve_count_epilogue<kModeStandard>(E, counts, d, st) : launch_sieve_count_epilogue<kModeLeftmost>(E, counts, d, st);
    else
        rc = mode == kModeStandard   ? (cp ? launch_sieve_epilogue<kModeStandard, true>(E, d, st) : launch_sieve_epilogue<kModeStandard, false>(E, d, st))
             : mode == kModeLeftmost ? (cp ? launch_sieve_epilogue<kModeLeftmost, true>(E, d, st) : launch_sieve_epilogue<kModeLeftmost, false>(E, d, st))
                                     : (cp ? launch_sieve_epilogue<kModeOverlap, true>(E, d, st) : launch_sieve_epilogue<kModeOverlap, false>(E, d, st));
    if (rc) return rc;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

// acb_count_non_overlapping (by_pattern = false: counts per haystack, written), acb_pattern_counts_non_overlapping
// (by_pattern: counts per pattern, added to), acb_pattern_hits (hits, dev_counts unused; either search) and
// acb_match_mask_non_overlapping (mb, dev_counts unused: the selection's bytes OR-ed into the mask)
int non_overlapping_counts(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                           int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                           uint64_t *dev_counts, void *stream, bool by_pattern, const HitRows *hits = nullptr, bool overlapping = false,
                           const acb_pattern_filter *filter = nullptr, const MaskBits *mb = nullptr) {
    if (!a || !dev_sieve || !dev_offsets || !plan || (!dev_counts && !hits && !mb) || (mb && !mb->mask) || (total_bytes && !dev_bytes))
        return fail(ACB_EINVAL, "null argument");
    if (int rc = check_ws(ws)) return rc;
    if (n_haystacks < 0 || n_haystacks > 0xfffffffell) return fail(ACB_EINVAL, "n_haystacks out of range (0 .. 2^32 - 2)");
    SieveFilter F;
    bool filtered;
    if (int rc = filter_view(a, filter, n_haystacks, F, filtered)) return rc;
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (scan larger inputs in windows)");
    if (overlapping && a->impl->hdr.match_kind != ACB_STANDARD) return unsupported_overlapping(a);
    acb_plan want;
    acb_plan_scan(a, dev_bytes, total_bytes, (uint64_t)n_haystacks, &want);
    if (want.n_segments != plan->n_segments || want.segment_bytes != plan->segment_bytes || want.n_units != plan->n_units ||
        want.task_bytes != plan->task_bytes)
        return fail(ACB_EINVAL, "plan does not match the arguments (call acb_plan_scan again)");
    SieveHeader sh;
    if (int rc = sieve_header(a, sh)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_haystacks == 0 || total_bytes == 0) {
        if (n_haystacks && !by_pattern && !hits && !mb) CUDA_OK(cudaMemsetAsync(dev_counts, 0, (uint64_t)n_haystacks * sizeof(uint64_t), st));
        zero_outputs_kernel<<<(unsigned)((n_haystacks + 256) / 256), 256, 0, st>>>(
            reinterpret_cast<unsigned long long *>(ws->dev_unit_offsets), reinterpret_cast<unsigned long long *>(ws->dev_match_offsets),
            n_haystacks, reinterpret_cast<unsigned long long *>(ws->dev_total));
        g_launches++;
        CUDA_OK(cudaGetLastError());
        return ACB_OK;
    }
    const int mode = overlapping ? kModeOverlap : a->impl->hdr.match_kind == ACB_STANDARD ? kModeStandard : kModeLeftmost;
    return sieve_list_scan(a, dev_sieve, Batch{dev_bytes, dev_offsets, n_haystacks}, total_bytes, mode, false, nullptr, plan, ws, d, st,
                           reinterpret_cast<unsigned long long *>(dev_counts), by_pattern, hits, filtered ? &F : nullptr, mb);
}

}  // namespace

extern "C" {

int acb_profile(const acb_automaton *a, const void *dev_image, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                int64_t n_haystacks, uint64_t total_bytes, int overlapping, uint32_t *dev_visits, void *stream) {
    if (!a || !dev_image || !dev_visits || !dev_offsets) return fail(ACB_EINVAL, "bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const ImageHeader &h = a->impl->hdr;
    CUDA_OK(cudaMemsetAsync(dev_visits, 0, uint64_t(h.n_states) * 4, st));
    if (n_haystacks < 1 || total_bytes == 0) return ACB_OK;
    Batch B{dev_bytes, dev_offsets, n_haystacks};
    int64_t n_samples = 256;
    if ((uint64_t)n_samples > total_bytes / 1024 + 1) n_samples = (int64_t)(total_bytes / 1024 + 1);
    const DevImage im = make_view(h, dev_image);
    const int restart = (!overlapping && h.match_kind == ACB_STANDARD) ? 1 : 0;
    profile_kernel<<<(unsigned)((n_samples + 127) / 128), 128, 0, st>>>(im, B, dev_visits, n_samples, 1024, restart);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_select_non_overlapping(const acb_automaton *a, const int64_t *dev_rows, uint64_t n_rows, int64_t *dev_out, uint64_t *dev_count,
                                void *stream) {
    if (!a || !dev_out || !dev_count || (n_rows && !dev_rows)) return fail(ACB_EINVAL, "null argument");
    const ImageHeader &h = a->impl->hdr;
    const int kind = (int)h.match_kind;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    select_rows_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const long long *>(dev_rows), n_rows, kind == ACB_STANDARD ? kModeStandard : kModeLeftmost,
                                         kind == ACB_LEFTMOST_LONGEST ? 1 : 0, (long long)h.max_pat_len, reinterpret_cast<long long *>(dev_out),
                                         reinterpret_cast<unsigned long long *>(dev_count));
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_any_match_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                           int64_t n_haystacks, uint64_t total_bytes, uint8_t *dev_flags, uint64_t *dev_scratch,
                           const acb_pattern_filter *filter, void *stream) {
    if (!dev_flags) return fail(ACB_EINVAL, "null argument");
    return sieve_early_scan(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_flags, dev_scratch, stream, kSieveAny, filter);
}

int acb_any_match(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                  int64_t n_haystacks, uint64_t total_bytes, uint8_t *dev_flags, uint64_t *dev_scratch, void *stream) {
    return acb_any_match_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_flags, dev_scratch, nullptr, stream);
}

int acb_find_first_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                            int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_keys, uint64_t *dev_scratch,
                            const acb_pattern_filter *filter, void *stream) {
    if (!dev_keys) return fail(ACB_EINVAL, "null argument");
    if (!a) return fail(ACB_EINVAL, "null argument");
    return sieve_early_scan(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_keys, dev_scratch, stream,
                            kSieveFirst + (int)a->impl->hdr.match_kind, filter);
}

int acb_find_first(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_keys, uint64_t *dev_scratch, void *stream) {
    return acb_find_first_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_keys, dev_scratch, nullptr, stream);
}

int acb_count_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_counts, uint64_t *dev_scratch,
                                   const acb_pattern_filter *filter, void *stream) {
    if (!dev_counts) return fail(ACB_EINVAL, "null argument");
    return sieve_early_scan(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_counts, dev_scratch, stream, kSieveCount, filter);
}

int acb_count_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                          int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_counts, uint64_t *dev_scratch, void *stream) {
    return acb_count_overlapping_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_counts, dev_scratch, nullptr, stream);
}

int acb_count_non_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                       int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                       uint64_t *dev_counts, const acb_pattern_filter *filter, void *stream) {
    return non_overlapping_counts(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, dev_counts, stream, false, nullptr,
                                  false, filter);
}

int acb_count_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                              int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                              uint64_t *dev_counts, void *stream) {
    return acb_count_non_overlapping_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, dev_counts, nullptr, stream);
}

int acb_pattern_counts_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, uint64_t *dev_pattern_counts, uint64_t *dev_scratch,
                                   void *stream) {
    if (!dev_pattern_counts) return fail(ACB_EINVAL, "null argument");
    return sieve_early_scan(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_pattern_counts, dev_scratch, stream,
                            kSievePatterns);
}

int acb_pattern_counts_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                       int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                       uint64_t *dev_pattern_counts, void *stream) {
    return non_overlapping_counts(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, dev_pattern_counts, stream, true);
}

uint64_t acb_pattern_hit_row_words(uint64_t n_patterns) { return acb::hit_row_words(n_patterns); }

int acb_pattern_hits(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                     int64_t n_haystacks, uint64_t total_bytes, int overlapping, const acb_plan *plan, const acb_workspace *ws,
                     uint32_t *dev_rows, uint64_t row_words, void *stream) {
    if (!a || (row_words && !dev_rows)) return fail(ACB_EINVAL, "null argument");
    if (reinterpret_cast<uintptr_t>(dev_rows) & 7u) return fail(ACB_EINVAL, "dev_rows must be 8-byte aligned");
    if (overlapping != 0 && overlapping != 1) return fail(ACB_EINVAL, "overlapping must be 0 or 1");
    const HitRows hits{dev_rows, row_words, (uint32_t)a->impl->hdr.n_patterns};
    return non_overlapping_counts(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, nullptr, stream, false, &hits,
                                  overlapping != 0);
}

int acb_match_mask_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                        int64_t n_haystacks, uint64_t total_bytes, uint32_t *dev_mask, uint64_t bit_base,
                                        uint64_t *dev_scratch, const acb_pattern_filter *filter, void *stream) {
    if (!dev_mask) return fail(ACB_EINVAL, "null argument");
    return sieve_early_scan(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_mask, dev_scratch, stream, kSieveCover, filter,
                            bit_base);
}

int acb_match_mask_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                               int64_t n_haystacks, uint64_t total_bytes, uint32_t *dev_mask, uint64_t bit_base, uint64_t *dev_scratch,
                               void *stream) {
    return acb_match_mask_overlapping_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, dev_mask, bit_base, dev_scratch,
                                               nullptr, stream);
}

int acb_match_mask_non_overlapping_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes,
                                            const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan,
                                            const acb_workspace *ws, uint32_t *dev_mask, uint64_t bit_base,
                                            const acb_pattern_filter *filter, void *stream) {
    if (!dev_mask) return fail(ACB_EINVAL, "null argument");
    const MaskBits mb{dev_mask, bit_base};
    return non_overlapping_counts(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, nullptr, stream, false, nullptr,
                                  false, filter, &mb);
}

int acb_match_mask_non_overlapping(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                   int64_t n_haystacks, uint64_t total_bytes, const acb_plan *plan, const acb_workspace *ws,
                                   uint32_t *dev_mask, uint64_t bit_base, void *stream) {
    return acb_match_mask_non_overlapping_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, plan, ws, dev_mask, bit_base,
                                                   nullptr, stream);
}

int acb_mask_rows(const void *dev_rows, int row_bytes, uint64_t n_rows, const int64_t *dev_offsets, int64_t n_haystacks, uint32_t *dev_mask,
                  uint64_t bit_base, void *stream) {
    if (!dev_mask || !dev_offsets || (n_rows && !dev_rows)) return fail(ACB_EINVAL, "null argument");
    if (row_bytes != 4 && row_bytes != 8) return fail(ACB_EINVAL, "row_bytes must be 4 (acb_match records) or 8 (int64 rows)");
    if (n_haystacks < 0 || n_haystacks > 0xfffffffell) return fail(ACB_EINVAL, "n_haystacks out of range (0 .. 2^32 - 2)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_rows == 0 || n_haystacks == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint64_t blocks = (n_rows + 255) / 256;
    if (blocks > 16ull * d.sms) blocks = 16ull * d.sms;  // grid-stride beyond that
    if (row_bytes == 4)
        mask_rows_kernel<int32_t><<<(unsigned)blocks, 256, 0, st>>>(static_cast<const int32_t *>(dev_rows), n_rows, dev_offsets, n_haystacks,
                                                                    dev_mask, bit_base);
    else
        mask_rows_kernel<long long><<<(unsigned)blocks, 256, 0, st>>>(static_cast<const long long *>(dev_rows), n_rows, dev_offsets, n_haystacks,
                                                                      dev_mask, bit_base);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_mask_unpack(const uint32_t *dev_mask, uint64_t bit_base, uint64_t stride, uint64_t n, uint8_t *dev_out, void *stream) {
    if (n && (!dev_mask || !dev_out)) return fail(ACB_EINVAL, "null argument");
    if (stride == 0) return fail(ACB_EINVAL, "stride must be at least 1");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint64_t blocks = (n + 256 * 16 - 1) / (256 * 16);
    if (blocks > 16ull * d.sms) blocks = 16ull * d.sms;  // grid-stride beyond that
    mask_unpack_kernel<<<(unsigned)blocks, 256, 0, st>>>(dev_mask, bit_base, stride, n, dev_out);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_count_rows(const acb_automaton *a, const int64_t *dev_rows, uint64_t n_rows, uint64_t *dev_scratch, uint64_t *dev_count,
                   void *stream) {
    if (!a || !dev_count || (n_rows && (!dev_rows || !dev_scratch))) return fail(ACB_EINVAL, "null argument");
    if (n_rows >= 0xffffffffull) return fail(ACB_EINVAL, "n_rows out of range (0 .. 2^32 - 2)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_rows == 0) {
        CUDA_OK(cudaMemsetAsync(dev_count, 0, sizeof(uint64_t), st));
        return ACB_OK;
    }
    const ImageHeader &h = a->impl->hdr;
    const long long *rows = reinterpret_cast<const long long *>(dev_rows);
    unsigned long long n = n_rows;
    int mode = h.match_kind == ACB_STANDARD ? kModeStandard : kModeLeftmost;
    int longest = h.match_kind == ACB_LEFTMOST_LONGEST ? 1 : 0;
    long long max_len = (long long)h.max_pat_len;
    uint4 *pairs = reinterpret_cast<uint4 *>(dev_scratch);
    unsigned long long *count = reinterpret_cast<unsigned long long *>(dev_count);
    void *args[] = {&rows, &n, &mode, &longest, &max_len, &pairs, &count};
    if (int rc = launch_cooperative(reinterpret_cast<const void *>(count_rows_kernel), args, d, st)) return rc;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_first_rows_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                            int64_t n_haystacks, const uint64_t *dev_keys, int64_t *dev_rows, const acb_pattern_filter *filter, void *stream) {
    if (!a || !dev_sieve || !dev_offsets || !dev_keys || !dev_rows) return fail(ACB_EINVAL, "null argument");
    if (n_haystacks < 0 || n_haystacks > 0xfffffffell) return fail(ACB_EINVAL, "n_haystacks out of range (0 .. 2^32 - 2)");
    SieveFilter F;
    bool filtered;
    if (int rc = filter_view(a, filter, n_haystacks, F, filtered)) return rc;
    SieveHeader sh;
    if (int rc = sieve_header(a, sh)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_haystacks == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int64_t blocks = (n_haystacks + 127) / 128;
    if (blocks > 16ll * d.sms) blocks = 16ll * d.sms;  // grid-stride beyond that
    const uint32_t *pat_len = reinterpret_cast<const uint32_t *>(static_cast<const uint8_t *>(dev_sieve) + sh.off_pat_len);
    if (filtered)
        first_rows_filtered_kernel<<<(unsigned)blocks, 128, 0, st>>>(make_sieve_view(sh, dev_sieve), pat_len, Batch{dev_bytes, dev_offsets, n_haystacks},
                                                                     reinterpret_cast<const unsigned long long *>(dev_keys),
                                                                     reinterpret_cast<long long *>(dev_rows), (int)a->impl->hdr.match_kind, F);
    else
        first_rows_kernel<<<(unsigned)blocks, 128, 0, st>>>(make_sieve_view(sh, dev_sieve), pat_len, Batch{dev_bytes, dev_offsets, n_haystacks},
                                                            reinterpret_cast<const unsigned long long *>(dev_keys),
                                                            reinterpret_cast<long long *>(dev_rows), (int)a->impl->hdr.match_kind);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_first_rows(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                   int64_t n_haystacks, const uint64_t *dev_keys, int64_t *dev_rows, void *stream) {
    return acb_first_rows_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_haystacks, dev_keys, dev_rows, nullptr, stream);
}

int acb_rows_to_codepoints(const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes,
                           const int64_t *dev_rows, int64_t *dev_cp_rows, void *stream) {
    if (!dev_offsets || !dev_rows || !dev_cp_rows || (total_bytes && !dev_bytes)) return fail(ACB_EINVAL, "null argument");
    if (dev_rows == dev_cp_rows) return fail(ACB_EINVAL, "dev_cp_rows must not be dev_rows");
    if (n_haystacks < 0) return fail(ACB_EINVAL, "n_haystacks out of range");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_haystacks == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemcpyAsync(dev_cp_rows, dev_rows, (uint64_t)n_haystacks * 3 * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    if (total_bytes == 0) return ACB_OK;
    const int64_t tiles = (int64_t)((total_bytes + kCpTile - 1) / kCpTile);
    int64_t blocks = (tiles + 7) / 8;  // 8 warps per block, a tile per warp
    if (blocks > 8ll * d.sms) blocks = 8ll * d.sms;  // grid-stride beyond that
    rows_to_codepoints_kernel<<<(unsigned)blocks, 256, 0, st>>>(Batch{dev_bytes, dev_offsets, n_haystacks}, (int64_t)total_bytes,
                                                                reinterpret_cast<const long long *>(dev_rows),
                                                                reinterpret_cast<long long *>(dev_cp_rows));
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

}  // extern "C"

template <typename T>
static void tokens_launch(const void *ids, uint64_t n, uint8_t *out, uint64_t *bad, int sms, cudaStream_t st) {
    const bool vec = (reinterpret_cast<uintptr_t>(ids) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out) & 3u) == 0;
    const uint64_t items = vec ? n / kTokGroup + n % kTokGroup : n;   // groups, then the tail's ids one per thread
    uint64_t blocks = (items + kTokThreads - 1) / kTokThreads;
    if (blocks > 8ull * (uint64_t)sms) blocks = 8ull * (uint64_t)sms;  // a full SM of 256-thread blocks, grid-stride beyond
    if (blocks < 1) blocks = 1;
    const T *p = static_cast<const T *>(ids);
    auto *b = reinterpret_cast<unsigned long long *>(bad);
    if (vec)
        tokens_encode_kernel<T, true><<<(unsigned)blocks, kTokThreads, 0, st>>>(p, n, out, b);
    else
        tokens_encode_kernel<T, false><<<(unsigned)blocks, kTokThreads, 0, st>>>(p, n, out, b);
    g_launches++;
}

extern "C" {

static int tokens_check(const void *ids, int token_bytes, uint64_t n, const uint8_t *out, const uint64_t *bad) {
    if (token_bytes != 2 && token_bytes != 4 && token_bytes != 8) return fail(ACB_EINVAL, "token_bytes must be 2, 4 or 8");
    if (n >= (1ull << 60)) return fail(ACB_EINVAL, "n_tokens out of range (0 .. 2^60 - 1)");
    if (!bad || (n && (!ids || !out))) return fail(ACB_EINVAL, "null argument");
    return ACB_OK;
}

int acb_tokens_encode(const void *dev_tokens, int token_bytes, uint64_t n_tokens, uint8_t *dev_out, uint64_t *dev_bad, void *stream) {
    if (int rc = tokens_check(dev_tokens, token_bytes, n_tokens, dev_out, dev_bad)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_tokens == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (token_bytes == 2) tokens_launch<uint16_t>(dev_tokens, n_tokens, dev_out, dev_bad, d.sms, st);
    else if (token_bytes == 4) tokens_launch<int32_t>(dev_tokens, n_tokens, dev_out, dev_bad, d.sms, st);
    else tokens_launch<int64_t>(dev_tokens, n_tokens, dev_out, dev_bad, d.sms, st);
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_tokens_encode_host(const void *host_tokens, int token_bytes, uint64_t n_tokens, uint8_t *host_out, uint64_t *host_bad) {
    if (int rc = tokens_check(host_tokens, token_bytes, n_tokens, host_out, host_bad)) return rc;
    if (token_bytes == 2) token_encode_host(static_cast<const uint16_t *>(host_tokens), n_tokens, host_out, host_bad);
    else if (token_bytes == 4) token_encode_host(static_cast<const int32_t *>(host_tokens), n_tokens, host_out, host_bad);
    else token_encode_host(static_cast<const int64_t *>(host_tokens), n_tokens, host_out, host_bad);
    return ACB_OK;
}

int acb_pack_gather_block(const uint64_t *dev_total, const acb_match *dev_out, uint32_t hay_base, uint64_t cap, void *dev_block, void *stream) {
    if (!dev_total || !dev_out || !dev_block) return fail(ACB_EINVAL, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    unsigned blocks = (unsigned)((cap + 255) / 256);
    if (blocks > 2u * (unsigned)d.sms) blocks = 2u * (unsigned)d.sms;  // two blocks per SM, grid-stride beyond that
    if (blocks < 1) blocks = 1;
    pack_gather_block_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const unsigned long long *>(dev_total), dev_out, hay_base, cap,
                                                     reinterpret_cast<uint4 *>(dev_block));
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_scan_batch_filtered(const acb_automaton *a, const void *dev_image, const void *dev_hot, const acb_hot_desc *hot_desc,
                            const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks,
                            uint64_t total_bytes, int overlapping, int codepoints, const acb_plan *plan, const acb_workspace *ws,
                            const acb_pattern_filter *filter, void *stream) {
    if (!a || !dev_image || !dev_offsets || n_haystacks < 0 || !plan) return fail(ACB_EINVAL, "bad argument");
    if (n_haystacks > 0xfffffffell) return fail(ACB_EINVAL, "too many haystacks in one batch");
    SieveFilter F;
    bool filtered;
    if (int rc = filter_view(a, filter, n_haystacks, F, filtered)) return rc;
    // the table images hold every pattern: a filtered scan always runs the sieve
    if (filtered && !dev_sieve) return fail(ACB_EINVAL, "a scan with pattern sets needs the sieve image");
    const ImageHeader &h = a->impl->hdr;
    const int kind = (int)h.match_kind;
    // overlapping == 2: the overlapping LIST, for any match kind -- the input of acb_select_non_overlapping; sieve only
    if (overlapping == 1 && kind != ACB_STANDARD)
        return fail(ACB_EUNSUPPORTED, std::string("match kind ") + (kind == ACB_LEFTMOST_FIRST ? "LeftmostFirst" : "LeftmostLongest") +
                                          " does not support overlapping searches");
    if (overlapping == 2 && !dev_sieve) return fail(ACB_EINVAL, "the overlapping list of a leftmost automaton needs the sieve image");
    int rc = check_ws(ws);
    if (rc) return rc;
    DeviceInfo d;
    if ((rc = device_info(d))) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int mode = overlapping ? kModeOverlap : (kind == ACB_STANDARD ? kModeStandard : kModeLeftmost);
    const bool cp = codepoints != 0;
    const DevImage im = make_view(h, dev_image);
    Batch B{dev_bytes, dev_offsets, n_haystacks};

    // the plan must be the one acb_plan_scan gives for these arguments (it sizes the workspace)
    acb_plan want;
    acb_plan_scan(a, dev_bytes, total_bytes, (uint64_t)n_haystacks, &want);
    if (want.n_segments != plan->n_segments || want.segment_bytes != plan->segment_bytes || want.n_units != plan->n_units ||
        want.task_bytes != plan->task_bytes)
        return fail(ACB_EINVAL, "plan does not match the arguments (call acb_plan_scan again)");

    unsigned long long *totals = reinterpret_cast<unsigned long long *>(ws->dev_total);
    unsigned int *task_counter = reinterpret_cast<unsigned int *>(ws->dev_scratch);
    Sink out;
    out.raw = ws->dev_raw;
    out.raw_seq = ws->dev_raw_seq;
    out.raw_unit = ws->dev_raw_unit;
    out.raw_aux = ws->dev_raw_aux;
    out.cap = ws->raw_capacity;
    out.unit_counts = ws->dev_unit_counts;
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(ws->dev_scratch);  // zero between scans (see kAcc*)
    out.raw_total = acc + kAccRaw;

    unsigned long long *unit_offsets = reinterpret_cast<unsigned long long *>(ws->dev_unit_offsets);
    unsigned long long *match_offsets = reinterpret_cast<unsigned long long *>(ws->dev_match_offsets);
    if (n_haystacks == 0 || total_bytes == 0) {
        zero_outputs_kernel<<<(unsigned)((n_haystacks + 256) / 256), 256, 0, st>>>(unit_offsets, match_offsets, n_haystacks, totals);
        g_launches++;
        CUDA_OK(cudaGetLastError());
        return ACB_OK;
    }

    int kernel = g_tuning.kernel;
    if (kernel == 0) kernel = dev_sieve ? 5 : 2;  // the caller uploads a sieve image when it wants the position-parallel scan
    if (overlapping == 2 || filtered) kernel = 5;
    // the caller's profile says the hot rows do not cover this data: scan from the image in global memory / L2
    if (kernel == 2 && g_tuning.kernel == 0 && hot_desc && (hot_desc->reserved & 1u)) kernel = 4;
    if (kernel == 5 && !dev_sieve) return fail(ACB_EINVAL, "the sieve kernel needs a sieve image (acb_sieve_build / acb_sieve_write)");
    if ((!dev_hot || !hot_desc) && kernel != 4 && kernel != 5) kernel = 1;  // no hot image: the plain kernel (one thread per haystack)
    if (kernel == 5)
        return sieve_list_scan(a, dev_sieve, B, total_bytes, mode, cp, im.pat_cplen, plan, ws, d, st, nullptr, false, nullptr,
                               filtered ? &F : nullptr);
    const bool segments = kernel == 2 || kernel == 3 || kernel == 4;
    const int per_lane = kernel == 3 ? 2 : 1;  // segments per lane of the staged kernel (3: two interleaved chains)
    SegPlan P{};

    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (g_timing) {
        CUDA_OK(cudaEventCreate(&ev0));
        CUDA_OK(cudaEventCreate(&ev1));
        CUDA_OK(cudaEventRecord(ev0, st));
    }
#define ACB_DISPATCH(FN, ...)                                                                                      \
    (mode == kModeStandard   ? (cp ? FN<kModeStandard, true>(__VA_ARGS__) : FN<kModeStandard, false>(__VA_ARGS__)) \
     : mode == kModeLeftmost ? (cp ? FN<kModeLeftmost, true>(__VA_ARGS__) : FN<kModeLeftmost, false>(__VA_ARGS__)) \
                             : (cp ? FN<kModeOverlap, true>(__VA_ARGS__) : FN<kModeOverlap, false>(__VA_ARGS__)))
    if (segments) {
        // the grid is anchored at the 64-byte aligned address at or before the buffer; the stream
        // bounds (offsets[0], offsets[n]) live on the device and are read by the kernels
        P.origin = -(int64_t)(reinterpret_cast<uintptr_t>(dev_bytes) & 63u);
        P.seg_bytes = plan->segment_bytes;
        P.warm = plan->warm_bytes;
        P.n_segments = (int64_t)plan->n_segments;
        P.lane_stride = plan->lane_stride;
        P.avg_len = n_haystacks > 0 ? total_bytes / (uint64_t)n_haystacks : 0;
    }
    // segment summaries: seg_info holds 32 bytes per segment -- SegRest[n] | keys u64[n] | code points: cont tails u32[n];
    // the counts take unit_counts: slot 1 [0, n), slot 0 [n, 2n)
    SegOut seg_out{};
    if (segments) {
        uint8_t *si = static_cast<uint8_t *>(ws->dev_seg_info);
        const uint64_t n = plan->n_segments;
        seg_out.rest = reinterpret_cast<SegRest *>(si);
        seg_out.key = reinterpret_cast<uint2 *>(si + 16 * n);
        seg_out.cont_tail = cp ? reinterpret_cast<uint32_t *>(si + 24 * n) : nullptr;
        seg_out.count = ws->dev_unit_counts;
        seg_out.count0 = ws->dev_unit_counts + n;
        seg_out.cont_far = reinterpret_cast<unsigned int *>(acc + kAccContFar);
    }
    if (kernel == 4) {
        rc = ACB_DISPATCH(launch_global, im, B, P, out, seg_out, d, st);
        if (rc) return rc;
        CUDA_OK(cudaGetLastError());
        if (ev1) {
            CUDA_OK(cudaEventRecord(ev1, st));
            g_timing_events.emplace_back(ev0, ev1);
        }
    } else if (segments) {
        DevHot hot;
        if ((rc = make_hot_view(a, dev_hot, *hot_desc, hot))) return rc;
        // the byte-indexed table is used when it exists and every row the profile saw fits on chip
        uint32_t fit128 = ascii_rows_that_fit(d);
        if (fit128 > hot.n_rows128) fit128 = hot.n_rows128;
        if (g_tuning.hot_rows > 0 && (uint32_t)g_tuning.hot_rows < fit128) fit128 = (uint32_t)g_tuning.hot_rows;
        // Byte-indexed (128-wide) rows make the transition two instructions per byte (IDP4A + LDS) instead of four,
        // but they are 256 bytes each (only ~230 fit below 64 KB), and on the config-2 text the kernel is bound by
        // the arrival of its staged bytes, not by the chain (on an H100 the warps wait for their next chunk ~60 % of
        // the time; DESIGN.md §6), so it is no faster than the compact table.
        // Opt-in (tuning.table = 2), one segment per lane only (two per lane leave too little room for the rows).
        const bool ascii = g_tuning.table == 2 && fit128 > 0 && per_lane == 1;
        rc = ACB_DISPATCH(launch_staged_cols, h, im, hot, B, P, out, seg_out, d, task_counter, acc + kAccGroups, st, ascii, per_lane);
        if (rc) return rc;
        CUDA_OK(cudaGetLastError());
        if (ev1) {
            CUDA_OK(cudaEventRecord(ev1, st));
            g_timing_events.emplace_back(ev0, ev1);
        }
    } else {
        rc = ACB_DISPATCH(launch_plain, im, B, out, d, st);
        if (rc) return rc;
        CUDA_OK(cudaGetLastError());
        if (ev1) {
            CUDA_OK(cudaEventRecord(ev1, st));
            g_timing_events.emplace_back(ev0, ev1);
        }
    }
    // counts (+ repair) -> offsets -> ordered output -> per-haystack offsets: one cooperative kernel
    const uint64_t max_tiles = (plan->n_units + kScanTile - 1) / kScanTile;
    unsigned long long *tile_sums = acc + kAccWords;
    unsigned long long *cont_tiles = tile_sums + max_tiles + 1;
    unsigned long long *cont_cum = cont_tiles + max_tiles + 1;
    EpilogueArgs E;
    E.im = im;
    E.B = B;
    E.P = P;
    E.out = out;
    E.seg = seg_out;
    E.counts = ws->dev_unit_counts;
    E.n_items = segments ? plan->n_segments : (uint64_t)n_haystacks;
    E.masks = reinterpret_cast<uint8_t *>(acc + want.scratch_words - (plan->n_units / 64 + 2));  // the last words of the scratch
    E.tile_sums = tile_sums;
    E.unit_offsets = unit_offsets;
    E.cont_tiles = cont_tiles;
    E.cont_cum = cont_cum;
    E.totals = totals;
    E.acc = acc;
    E.raw = ws->dev_raw;
    E.raw_seq = ws->dev_raw_seq;
    E.raw_unit = ws->dev_raw_unit;
    E.raw_aux = ws->dev_raw_aux;
    E.raw_cap = ws->raw_capacity;
    E.pat_cplen = im.pat_cplen;
    E.out_buf = ws->dev_out;
    E.out_cap = ws->out_capacity;
    E.match_offsets = match_offsets;
    E.need_repair = task_counter + 1;
    E.do_repair = (segments && mode != kModeOverlap) ? 1 : 0;
    rc = ACB_DISPATCH(launch_epilogue, E, d, st);
#undef ACB_DISPATCH
    if (rc) return rc;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_scan_batch(const acb_automaton *a, const void *dev_image, const void *dev_hot, const acb_hot_desc *hot_desc,
                   const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_haystacks, uint64_t total_bytes,
                   int overlapping, int codepoints, const acb_plan *plan, const acb_workspace *ws, void *stream) {
    return acb_scan_batch_filtered(a, dev_image, dev_hot, hot_desc, dev_sieve, dev_bytes, dev_offsets, n_haystacks, total_bytes, overlapping,
                                   codepoints, plan, ws, nullptr, stream);
}

int acb_stream_seams(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                     const int64_t *dev_carry, const uint8_t *dev_tail, uint8_t *dev_seam_bytes, int64_t *dev_seam_offsets, void *stream) {
    if (!a || !dev_offsets || !dev_carry || !dev_seam_offsets || (total_bytes && !dev_bytes)) return fail(ACB_EINVAL, "null argument");
    const uint32_t halo = a->impl->hdr.max_pat_len ? a->impl->hdr.max_pat_len - 1 : 0;
    if (halo && (!dev_tail || !dev_seam_bytes)) return fail(ACB_EINVAL, "null argument");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (feed larger data in more chunks)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_streams == 0) {
        CUDA_OK(cudaMemsetAsync(dev_seam_offsets, 0, sizeof(int64_t), st));
        return ACB_OK;
    }
    int64_t blocks = (n_streams + 255) / 256;
    if (blocks > 8ll * d.sms) blocks = 8ll * d.sms;
    stream_seam_lengths_kernel<<<(unsigned)blocks, 256, 0, st>>>(dev_offsets, n_streams, dev_carry, halo, dev_seam_offsets);
    stream_prefix_kernel<<<1, kScanThreads, 0, st>>>(dev_seam_offsets, n_streams);
    int64_t fill_blocks = (n_streams + 7) / 8;  // a warp per stream
    if (fill_blocks > 16ll * d.sms) fill_blocks = 16ll * d.sms;
    if (halo)
        stream_seam_fill_kernel<<<(unsigned)fill_blocks, 256, 0, st>>>(dev_bytes, dev_offsets, n_streams, dev_carry, dev_tail, halo,
                                                                       dev_seam_offsets, dev_seam_bytes);
    g_launches += halo ? 3 : 2;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_resolve(const acb_automaton *a, const void *dev_image, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams,
                       uint64_t total_bytes, const uint8_t *dev_last, int overlapping, int codepoints, int64_t *dev_carry, uint8_t *dev_tail,
                       const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, const acb_match *dev_seam_list,
                       const uint64_t *dev_seam_match_offsets, const acb_match *dev_chunk_list, const uint64_t *dev_chunk_match_offsets,
                       int64_t *dev_scratch, int64_t *dev_rows, int64_t *dev_row_offsets, void *stream) {
    if (!a || !dev_offsets || !dev_carry || !dev_seam_offsets || !dev_seam_list || !dev_seam_match_offsets || !dev_chunk_list ||
        !dev_chunk_match_offsets || !dev_scratch || !dev_rows || !dev_row_offsets || (total_bytes && !dev_bytes))
        return fail(ACB_EINVAL, "null argument");
    const ImageHeader &h = a->impl->hdr;
    const int kind = (int)h.match_kind;
    if (overlapping != 0 && overlapping != 1) return fail(ACB_EINVAL, "overlapping must be 0 or 1");
    if (overlapping && kind != ACB_STANDARD)
        return fail(ACB_EUNSUPPORTED, std::string("match kind ") + (kind == ACB_LEFTMOST_FIRST ? "LeftmostFirst" : "LeftmostLongest") +
                                          " does not support overlapping searches");
    const uint32_t halo = h.max_pat_len ? h.max_pat_len - 1 : 0;
    if (halo && (!dev_tail || !dev_seam_bytes)) return fail(ACB_EINVAL, "null argument");
    if (codepoints && !dev_image) return fail(ACB_EINVAL, "code points need the device image (pattern lengths in code points)");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (feed larger data in more chunks)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemsetAsync(dev_scratch, 0, 2 * sizeof(uint64_t), st));
    if (n_streams == 0) {
        CUDA_OK(cudaMemsetAsync(dev_row_offsets, 0, sizeof(int64_t), st));
        return ACB_OK;
    }
    StreamArgs A;
    A.B = Batch{dev_bytes, dev_offsets, n_streams};
    A.carry = dev_carry;
    A.tail = dev_tail;
    A.last = dev_last;
    A.seam = dev_seam_bytes;
    A.seam_offsets = dev_seam_offsets;
    A.seam_list = reinterpret_cast<const uint4 *>(dev_seam_list);
    A.chunk_list = reinterpret_cast<const uint4 *>(dev_chunk_list);
    A.seam_mo = reinterpret_cast<const unsigned long long *>(dev_seam_match_offsets);
    A.chunk_mo = reinterpret_cast<const unsigned long long *>(dev_chunk_match_offsets);
    A.stats = reinterpret_cast<unsigned long long *>(dev_scratch);
    A.cont_rows = reinterpret_cast<long long *>(dev_scratch + 2);
    A.cont_cp = reinterpret_cast<long long *>(dev_scratch + 2 + 3 * n_streams);
    A.staged = reinterpret_cast<long long *>(dev_scratch + 2 + 6 * n_streams);
    A.row_offsets = dev_row_offsets;
    A.rows = reinterpret_cast<long long *>(dev_rows);
    A.pat_cplen = codepoints ? make_view(h, dev_image).pat_cplen : nullptr;
    A.halo = halo;
    A.mode = overlapping ? kModeOverlap : (kind == ACB_STANDARD ? kModeStandard : kModeLeftmost);
    A.longest = kind == ACB_LEFTMOST_LONGEST ? 1 : 0;
    A.codepoints = codepoints ? 1 : 0;
    int64_t blocks = (n_streams + 127) / 128;
    if (blocks > 16ll * d.sms) blocks = 16ll * d.sms;
    if (A.mode == kModeOverlap)
        stream_select_kernel<kModeOverlap><<<(unsigned)blocks, 128, 0, st>>>(A);
    else if (A.mode == kModeStandard)
        stream_select_kernel<kModeStandard><<<(unsigned)blocks, 128, 0, st>>>(A);
    else
        stream_select_kernel<kModeLeftmost><<<(unsigned)blocks, 128, 0, st>>>(A);
    stream_prefix_kernel<<<1, kScanThreads, 0, st>>>(dev_row_offsets, n_streams);
    g_launches += 2;
    CUDA_OK(cudaGetLastError());
    if (codepoints) {  // continuation bytes of each chunk before its new tail, counted on the whole grid
        if (int rc = acb_rows_to_codepoints(dev_bytes, dev_offsets, n_streams, total_bytes, reinterpret_cast<const int64_t *>(A.cont_rows),
                                            reinterpret_cast<int64_t *>(A.cont_cp), stream))
            return rc;
    }
    if (!codepoints) {  // the row count is on the device only: a grid of 8 blocks per SM, grid-stride over the rows
        stream_rows_kernel<<<(unsigned)(8 * d.sms), 256, 0, st>>>(A);
        g_launches++;
    }
    int64_t emit_blocks = (n_streams + 7) / 8;  // a warp per stream
    if (emit_blocks > 16ll * d.sms) emit_blocks = 16ll * d.sms;
    stream_emit_kernel<<<(unsigned)emit_blocks, 256, 0, st>>>(A);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_advance(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                       const uint8_t *dev_last, int codepoints, int64_t *dev_carry, uint8_t *dev_tail, const uint8_t *dev_seam_bytes,
                       const int64_t *dev_seam_offsets, int64_t *dev_scratch, void *stream) {
    if (!a || !dev_offsets || !dev_carry || !dev_seam_offsets || (total_bytes && !dev_bytes) || (codepoints && !dev_scratch))
        return fail(ACB_EINVAL, "null argument");
    const uint32_t halo = a->impl->hdr.max_pat_len ? a->impl->hdr.max_pat_len - 1 : 0;
    if (halo && (!dev_tail || !dev_seam_bytes)) return fail(ACB_EINVAL, "null argument");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (feed larger data in more chunks)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_streams == 0) return ACB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    StreamArgs A = {};
    A.B = Batch{dev_bytes, dev_offsets, n_streams};
    A.carry = dev_carry;
    A.tail = dev_tail;
    A.last = dev_last;
    A.seam = dev_seam_bytes;
    A.seam_offsets = dev_seam_offsets;
    A.halo = halo;
    A.codepoints = codepoints ? 1 : 0;
    if (codepoints) {  // continuation bytes of each chunk before its new tail, counted on the whole grid
        A.cont_rows = reinterpret_cast<long long *>(dev_scratch);
        A.cont_cp = reinterpret_cast<long long *>(dev_scratch + 3 * n_streams);
        int64_t blocks = (n_streams + 255) / 256;
        if (blocks > 8ll * d.sms) blocks = 8ll * d.sms;
        stream_cont_rows_kernel<<<(unsigned)blocks, 256, 0, st>>>(A);
        g_launches++;
        CUDA_OK(cudaGetLastError());
        if (int rc = acb_rows_to_codepoints(dev_bytes, dev_offsets, n_streams, total_bytes, reinterpret_cast<const int64_t *>(A.cont_rows),
                                            reinterpret_cast<int64_t *>(A.cont_cp), stream))
            return rc;
    }
    int64_t blocks = (n_streams + 7) / 8;  // a warp per stream
    if (blocks > 16ll * d.sms) blocks = 16ll * d.sms;
    stream_advance_kernel<<<(unsigned)blocks, 256, 0, st>>>(A);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_first_resolve_filtered(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                                      int64_t n_streams, uint64_t total_bytes, const uint8_t *dev_last, int codepoints, const int64_t *dev_carry,
                                      const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, uint64_t seam_buffer_bytes,
                                      uint64_t *dev_seam_keys, uint64_t *dev_chunk_keys, int64_t *dev_best, int64_t *dev_scratch,
                                      int64_t *dev_rows, const acb_pattern_filter *filter, void *stream) {
    if (!a || !dev_sieve || !dev_offsets || !dev_carry || !dev_seam_offsets || !dev_seam_keys || !dev_chunk_keys || !dev_best ||
        !dev_scratch || !dev_rows || (total_bytes && !dev_bytes) || (seam_buffer_bytes && !dev_seam_bytes))
        return fail(ACB_EINVAL, "null argument");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    {
        SieveFilter F;
        bool filtered;
        if (int rc = filter_view(a, filter, n_streams, F, filtered)) return rc;
    }
    if (total_bytes >= (1ull << 31) || seam_buffer_bytes >= (1ull << 31))
        return fail(ACB_EINVAL, "total_bytes and seam_buffer_bytes must be below 2^31 (feed larger data in more chunks)");
    SieveHeader sh;
    if (int rc = sieve_header(a, sh)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemsetAsync(dev_scratch, 0, 2 * sizeof(uint64_t), st));
    if (n_streams == 0) return ACB_OK;
    const int64_t n = n_streams;
    FirstArgs A;
    A.B = Batch{dev_bytes, dev_offsets, n};
    A.carry = dev_carry;
    A.last = dev_last;
    A.seam = dev_seam_bytes;
    A.seam_offsets = dev_seam_offsets;
    A.seam_keys = reinterpret_cast<unsigned long long *>(dev_seam_keys);
    A.chunk_keys = reinterpret_cast<unsigned long long *>(dev_chunk_keys);
    A.seam_rows = reinterpret_cast<long long *>(dev_scratch + 2);
    A.chunk_rows = reinterpret_cast<long long *>(dev_scratch + 2 + 3 * n);
    A.seam_cp = reinterpret_cast<long long *>(dev_scratch + 2 + 6 * n);
    A.chunk_cp = reinterpret_cast<long long *>(dev_scratch + 2 + 9 * n);
    A.best = reinterpret_cast<long long *>(dev_best);
    A.rows = reinterpret_cast<long long *>(dev_rows);
    A.stats = reinterpret_cast<unsigned long long *>(dev_scratch);
    A.max_len = a->impl->hdr.max_pat_len;
    A.kind = (int)a->impl->hdr.match_kind;
    A.codepoints = codepoints ? 1 : 0;
    int64_t blocks = (n + 127) / 128;
    if (blocks > 16ll * d.sms) blocks = 16ll * d.sms;
    stream_first_unmask_kernel<<<(unsigned)blocks, 128, 0, st>>>(A);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    const Batch seams{dev_seam_bytes, dev_seam_offsets, n};
    if (int rc = acb_first_rows_filtered(a, dev_sieve, seams.bytes, seams.offsets, n, dev_seam_keys, dev_scratch + 2, filter, stream)) return rc;
    if (int rc = acb_first_rows_filtered(a, dev_sieve, dev_bytes, dev_offsets, n, dev_chunk_keys, dev_scratch + 2 + 3 * n, filter, stream))
        return rc;
    if (codepoints) {
        if (int rc = acb_rows_to_codepoints(seams.bytes, seams.offsets, n, seam_buffer_bytes, dev_scratch + 2, dev_scratch + 2 + 6 * n, stream))
            return rc;
        if (int rc = acb_rows_to_codepoints(dev_bytes, dev_offsets, n, total_bytes, dev_scratch + 2 + 3 * n, dev_scratch + 2 + 9 * n, stream))
            return rc;
    }
    stream_first_resolve_kernel<<<(unsigned)blocks, 128, 0, st>>>(A);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_first_resolve(const acb_automaton *a, const void *dev_sieve, const uint8_t *dev_bytes, const int64_t *dev_offsets,
                             int64_t n_streams, uint64_t total_bytes, const uint8_t *dev_last, int codepoints, const int64_t *dev_carry,
                             const uint8_t *dev_seam_bytes, const int64_t *dev_seam_offsets, uint64_t seam_buffer_bytes,
                             uint64_t *dev_seam_keys, uint64_t *dev_chunk_keys, int64_t *dev_best, int64_t *dev_scratch, int64_t *dev_rows,
                             void *stream) {
    return acb_stream_first_resolve_filtered(a, dev_sieve, dev_bytes, dev_offsets, n_streams, total_bytes, dev_last, codepoints, dev_carry,
                                             dev_seam_bytes, dev_seam_offsets, seam_buffer_bytes, dev_seam_keys, dev_chunk_keys, dev_best,
                                             dev_scratch, dev_rows, nullptr, stream);
}

int acb_stream_count(const acb_automaton *a, const uint8_t *dev_bytes, const int64_t *dev_offsets, int64_t n_streams, uint64_t total_bytes,
                     const uint8_t *dev_last, int overlapping, int64_t *dev_carry, const int64_t *dev_seam_offsets,
                     const acb_match *dev_seam_list, const uint64_t *dev_seam_match_offsets, const acb_match *dev_chunk_list,
                     const uint64_t *dev_chunk_match_offsets, const uint64_t *dev_chunk_counts, int64_t *dev_running, int64_t *dev_counts,
                     int64_t *dev_scratch, uint64_t scratch_words, void *stream) {
    if (!a || !dev_offsets || !dev_carry || !dev_seam_offsets || !dev_seam_list || !dev_seam_match_offsets || !dev_running || !dev_counts ||
        !dev_scratch || (total_bytes && !dev_bytes))
        return fail(ACB_EINVAL, "null argument");
    if (overlapping != 0 && overlapping != 1) return fail(ACB_EINVAL, "overlapping must be 0 or 1");
    if (overlapping ? !dev_chunk_counts : (!dev_chunk_list || !dev_chunk_match_offsets)) return fail(ACB_EINVAL, "null argument");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    if (total_bytes >= (1ull << 31)) return fail(ACB_EINVAL, "total_bytes must be below 2^31 (feed larger data in more chunks)");
    const uint64_t need = overlapping ? 4 : 4 + 6 * (uint64_t)n_streams;
    if (scratch_words < need) return fail(ACB_EINVAL, "dev_scratch is too small");
    const ImageHeader &h = a->impl->hdr;
    const int kind = (int)h.match_kind;
    if (overlapping && kind != ACB_STANDARD) return unsupported_overlapping(a);
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemsetAsync(dev_scratch, 0, 4 * sizeof(uint64_t), st));
    if (n_streams == 0) return ACB_OK;
    CountArgs A = {};
    A.S.B = Batch{dev_bytes, dev_offsets, n_streams};
    A.S.carry = dev_carry;
    A.S.last = dev_last;
    A.S.seam_offsets = dev_seam_offsets;
    A.S.seam_list = reinterpret_cast<const uint4 *>(dev_seam_list);
    A.S.chunk_list = reinterpret_cast<const uint4 *>(dev_chunk_list);
    A.S.seam_mo = reinterpret_cast<const unsigned long long *>(dev_seam_match_offsets);
    A.S.chunk_mo = reinterpret_cast<const unsigned long long *>(dev_chunk_match_offsets);
    A.S.halo = h.max_pat_len ? h.max_pat_len - 1 : 0;
    A.S.mode = overlapping ? kModeOverlap : (kind == ACB_STANDARD ? kModeStandard : kModeLeftmost);
    A.S.longest = kind == ACB_LEFTMOST_LONGEST ? 1 : 0;
    A.chunk_counts = reinterpret_cast<const unsigned long long *>(dev_chunk_counts);
    A.running = reinterpret_cast<long long *>(dev_running);
    A.out = reinterpret_cast<long long *>(dev_counts);
    A.stats = reinterpret_cast<unsigned long long *>(dev_scratch);
    if (overlapping) {
        int64_t blocks = (n_streams + 127) / 128;
        if (blocks > 16ll * d.sms) blocks = 16ll * d.sms;
        stream_count_overlap_kernel<<<(unsigned)blocks, 128, 0, st>>>(A);
        g_launches++;
        CUDA_OK(cudaGetLastError());
        return ACB_OK;
    }
    // records of both lists: each pair takes two words, each mark half of one
    const uint64_t r_max = (scratch_words - need) / 4;
    A.per = reinterpret_cast<long long *>(dev_scratch + 4);
    A.long_list = reinterpret_cast<long long *>(dev_scratch + 4 + 4 * n_streams);
    A.pairs = reinterpret_cast<uint4 *>(dev_scratch + need);
    A.mark = reinterpret_cast<uint32_t *>(dev_scratch + need + 2 * r_max);
    void *args[] = {&A};
    const void *kern = A.S.mode == kModeStandard ? reinterpret_cast<const void *>(stream_count_kernel<kModeStandard>)
                                                 : reinterpret_cast<const void *>(stream_count_kernel<kModeLeftmost>);
    if (int rc = launch_cooperative(kern, args, d, st)) return rc;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_mask_rows(const int64_t *dev_offsets, int64_t n_streams, const int64_t *dev_carry_before, const int64_t *dev_seam_offsets,
                         const int64_t *dev_rows, const int64_t *dev_row_offsets, uint32_t *dev_chunk_mask, uint32_t *dev_seam_mask,
                         void *stream) {
    if (!dev_offsets || !dev_carry_before || !dev_seam_offsets || !dev_rows || !dev_row_offsets || !dev_chunk_mask || !dev_seam_mask)
        return fail(ACB_EINVAL, "null argument");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_streams == 0) return ACB_OK;
    MaskStreamArgs A = {};
    A.offsets = dev_offsets;
    A.n = n_streams;
    A.carry = dev_carry_before;
    A.seam_offsets = dev_seam_offsets;
    A.chunk_mask = dev_chunk_mask;
    A.seam_mask = dev_seam_mask;
    // the row count is on the device only: a grid of 8 blocks per SM, grid-stride over the rows
    stream_mask_rows_kernel<<<(unsigned)(8 * d.sms), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        A, reinterpret_cast<const long long *>(dev_rows), dev_row_offsets);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_stream_mask_emit(const acb_automaton *a, const int64_t *dev_offsets, int64_t n_streams, const uint8_t *dev_last, int overlapping,
                         uint64_t stride, const int64_t *dev_carry_before, const int64_t *dev_seam_offsets, const uint32_t *dev_chunk_mask,
                         const uint32_t *dev_seam_mask, const uint8_t *dev_held_in, uint8_t *dev_held_out, uint8_t *dev_flags,
                         int64_t *dev_flag_offsets, int64_t *dev_flag_starts, void *stream) {
    if (!a || !dev_offsets || !dev_carry_before || !dev_seam_offsets || !dev_chunk_mask || !dev_seam_mask || !dev_flags || !dev_flag_offsets ||
        !dev_flag_starts)
        return fail(ACB_EINVAL, "null argument");
    const uint32_t halo = a->impl->hdr.max_pat_len ? a->impl->hdr.max_pat_len - 1 : 0;
    if (halo && (!dev_held_in || !dev_held_out)) return fail(ACB_EINVAL, "null argument");
    if (halo && dev_held_in == dev_held_out) return fail(ACB_EINVAL, "dev_held_in and dev_held_out must be different buffers");
    if (overlapping != 0 && overlapping != 1) return fail(ACB_EINVAL, "overlapping must be 0 or 1");
    if (stride == 0 || stride > 0xffffffffull) return fail(ACB_EINVAL, "stride out of range (1 .. 2^32 - 1)");
    if (n_streams < 0 || n_streams > 0xfffffffell) return fail(ACB_EINVAL, "n_streams out of range (0 .. 2^32 - 2)");
    if (overlapping && (int)a->impl->hdr.match_kind != ACB_STANDARD) return unsupported_overlapping(a);
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_streams == 0) {
        CUDA_OK(cudaMemsetAsync(dev_flag_offsets, 0, sizeof(int64_t), st));
        return ACB_OK;
    }
    MaskStreamArgs A = {};
    A.offsets = dev_offsets;
    A.n = n_streams;
    A.carry = dev_carry_before;
    A.seam_offsets = dev_seam_offsets;
    A.last = dev_last;
    A.chunk_mask = const_cast<uint32_t *>(dev_chunk_mask);
    A.seam_mask = const_cast<uint32_t *>(dev_seam_mask);
    A.held_in = dev_held_in;
    A.held_out = dev_held_out;
    A.flags = dev_flags;
    A.flag_offsets = dev_flag_offsets;
    A.flag_starts = dev_flag_starts;
    A.stride = stride;
    A.halo = halo;
    A.overlapping = overlapping;
    int64_t blocks = (n_streams + 255) / 256;
    if (blocks > 8ll * d.sms) blocks = 8ll * d.sms;
    stream_mask_count_kernel<<<(unsigned)blocks, 256, 0, st>>>(A);
    stream_prefix_kernel<<<1, kScanThreads, 0, st>>>(dev_flag_offsets, n_streams);
    // the flag count is on the device only: a grid of 8 blocks per SM, grid-stride over the flags and the held bytes
    stream_mask_emit_kernel<<<(unsigned)(8 * d.sms), 256, 0, st>>>(A);
    g_launches += 3;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

}  // extern "C"

// ===========================================================================
// Completing tokens (completions.h, completions.cuh)
// ===========================================================================
template <typename T, typename L, int MODE, bool FILT>
static void completions_launch(const ComplView &V, const void *tokens, uint64_t n_tokens, const int64_t *offsets, int64_t n_rows,
                               const SieveFilter &F, void *logits, int64_t row_stride, int64_t vocab, float value, int64_t *out,
                               const int64_t *out_offsets, int sms, cudaStream_t st) {
    constexpr int64_t kWarps = kComplThreads / 32;
    int64_t blocks = (n_rows + kWarps - 1) / kWarps;
    if (blocks > 32ll * sms) blocks = 32ll * sms;   // grid-stride beyond that
    completions_kernel<T, L, MODE, FILT><<<(unsigned)blocks, kComplThreads, 0, st>>>(
        V, static_cast<const T *>(tokens), n_tokens, offsets, n_rows, F, static_cast<L *>(logits), row_stride, vocab, value, out, out_offsets);
}

template <typename L, int MODE>
static void completions_dispatch(int token_bytes, bool filt, const ComplView &V, const void *tokens, uint64_t n_tokens,
                                 const int64_t *offsets, int64_t n_rows, const SieveFilter &F, void *logits, int64_t row_stride,
                                 int64_t vocab, float value, int64_t *out, const int64_t *out_offsets, int sms, cudaStream_t st) {
#define ACB_COMPL_LAUNCH(T, FL) \
    completions_launch<T, L, MODE, FL>(V, tokens, n_tokens, offsets, n_rows, F, logits, row_stride, vocab, value, out, out_offsets, sms, st)
    if (token_bytes == 2) {
        if (filt) ACB_COMPL_LAUNCH(uint16_t, true); else ACB_COMPL_LAUNCH(uint16_t, false);
    } else if (token_bytes == 4) {
        if (filt) ACB_COMPL_LAUNCH(int32_t, true); else ACB_COMPL_LAUNCH(int32_t, false);
    } else {
        if (filt) ACB_COMPL_LAUNCH(int64_t, true); else ACB_COMPL_LAUNCH(int64_t, false);
    }
#undef ACB_COMPL_LAUNCH
}

extern "C" {

int acb_completions_build(acb_automaton *a, uint64_t *image_bytes) {
    if (!a || !image_bytes) return fail(ACB_EINVAL, "null argument");
    Automaton &A = *a->impl;
    std::lock_guard<std::mutex> lock(A.sieve_mutex);
    if (A.completions.empty()) {
        // the patterns must be in the token format: whole 3-byte groups, each some id's token_code
        const uint64_t n = A.hdr.n_patterns;
        std::vector<uint32_t> ids;
        std::vector<uint64_t> offs(n + 1, 0);
        ids.reserve(A.pat_blob.size() / ACB_TOKEN_BYTES);
        for (uint64_t i = 0; i < n; i++) {
            const uint64_t s = A.pat_offs[i], e = A.pat_offs[i + 1];
            if ((e - s) % ACB_TOKEN_BYTES) return fail(ACB_EINVAL, "pattern " + std::to_string(i) + " is not in the token format (length not a multiple of 3)");
            for (uint64_t k = s; k < e; k += ACB_TOKEN_BYTES) {
                uint32_t t;
                if (!token_decode(A.pat_blob[k], A.pat_blob[k + 1], A.pat_blob[k + 2], t))
                    return fail(ACB_EINVAL, "pattern " + std::to_string(i) + " is not in the token format (byte " + std::to_string(k - s) + ")");
                ids.push_back(t);
            }
            offs[i + 1] = ids.size();
        }
        try {
            completions_image_build(ids.data(), offs.data(), n, A.completions);
        } catch (const std::exception &e) {
            A.completions.clear();
            return fail(ACB_EBUILD, e.what());
        }
    }
    *image_bytes = A.completions.size();
    return ACB_OK;
}

int acb_completions_write(acb_automaton *a, void *host_dst, uint64_t dst_bytes) {
    if (!a || !host_dst) return fail(ACB_EINVAL, "null argument");
    Automaton &A = *a->impl;
    std::lock_guard<std::mutex> lock(A.sieve_mutex);
    if (A.completions.empty()) return fail(ACB_EINVAL, "acb_completions_build has not been called");
    if (dst_bytes < A.completions.size()) return fail(ACB_ECAPACITY, "completions image buffer too small");
    std::memcpy(host_dst, A.completions.data(), A.completions.size());
    return ACB_OK;
}

int acb_completions_describe(const void *host_image, acb_completions_desc *d) {
    const ComplHeader *h = static_cast<const ComplHeader *>(host_image);
    if (!h || !d || h->magic != kComplMagic) return fail(ACB_EINVAL, "not a completions image");
    d->nodes = h->n_nodes;
    d->entries = h->n_entries;
    d->depth = h->depth;
    d->max_last = h->max_last;
    return ACB_OK;
}

}  // extern "C"

// the checks every completions entry point makes, before any CUDA call; the host header and the filter view
static int completions_check(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                             const int64_t *dev_offsets, int64_t n_rows, const acb_pattern_filter *filter, ComplHeader &h,
                             SieveFilter &F, bool &filt) {
    if (!a || !dev_image || (n_tokens && !dev_tokens) || (n_rows && !dev_offsets)) return fail(ACB_EINVAL, "null argument");
    if (token_bytes != 2 && token_bytes != 4 && token_bytes != 8) return fail(ACB_EINVAL, "token_bytes must be 2, 4 or 8");
    if (n_tokens >= (1ull << 60)) return fail(ACB_EINVAL, "n_tokens must be below 2^60");
    if (n_rows < 0 || n_rows > 0xfffffffell) return fail(ACB_EINVAL, "n_rows out of range (0 .. 2^32 - 2)");
    {
        std::lock_guard<std::mutex> lock(a->impl->sieve_mutex);
        if (a->impl->completions.size() < sizeof(ComplHeader)) return fail(ACB_EINVAL, "acb_completions_build has not been called");
        std::memcpy(&h, a->impl->completions.data(), sizeof(h));
    }
    return filter_view(a, filter, n_rows, F, filt);
}

// the logits checks of the mask and bias modes: the pointer, the dtype code, V, the row stride, and V > max_last
static int completions_logits_check(const ComplHeader &h, int64_t n_rows, const void *dev_logits, int logits_dtype, int64_t row_stride,
                                    int64_t vocab) {
    if (n_rows && !dev_logits) return fail(ACB_EINVAL, "null argument");
    if (logits_dtype != ACB_LOGITS_F32 && logits_dtype != ACB_LOGITS_F16 && logits_dtype != ACB_LOGITS_BF16)
        return fail(ACB_EINVAL, "logits_dtype must be ACB_LOGITS_F32, ACB_LOGITS_F16 or ACB_LOGITS_BF16");
    if (vocab < 1 || vocab >= (1ll << 62)) return fail(ACB_EINVAL, "vocab out of range (1 .. 2^62 - 1)");
    if (row_stride < 0 || row_stride >= (1ll << 62)) return fail(ACB_EINVAL, "row_stride out of range (0 .. 2^62 - 1)");
    if (h.n_entries && (int64_t)h.max_last >= vocab)
        return fail(ACB_EINVAL, "vocab " + std::to_string(vocab) + " does not hold the largest completing id " + std::to_string(h.max_last));
    return ACB_OK;
}

static ComplView completions_view(const ComplHeader &h, const void *dev_image) {
    const uint8_t *b = static_cast<const uint8_t *>(dev_image);
    ComplView V;
    V.nodes = reinterpret_cast<const ComplNode *>(b + h.off_nodes);
    V.kid_tok = reinterpret_cast<const uint32_t *>(b + h.off_kid_tok);
    V.entries = reinterpret_cast<const ComplEntry *>(b + h.off_entries);
    V.depth = h.depth;
    return V;
}

extern "C" {

int acb_completions_count(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                          const int64_t *dev_offsets, int64_t n_rows, int64_t *dev_counts, const acb_pattern_filter *filter, void *stream) {
    ComplHeader h;
    SieveFilter F{};
    bool filt = false;
    if (int rc = completions_check(a, dev_image, dev_tokens, token_bytes, n_tokens, dev_offsets, n_rows, filter, h, F, filt)) return rc;
    if (n_rows && !dev_counts) return fail(ACB_EINVAL, "null argument");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_rows == 0) return ACB_OK;
    completions_dispatch<float, kComplCount>(token_bytes, filt, completions_view(h, dev_image), dev_tokens, n_tokens, dev_offsets, n_rows, F,
                                             nullptr, 0, 0, 0.f, dev_counts, nullptr, d.sms, static_cast<cudaStream_t>(stream));
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_completions_emit(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, const int64_t *dev_row_offsets, int64_t *dev_ids,
                         const acb_pattern_filter *filter, void *stream) {
    ComplHeader h;
    SieveFilter F{};
    bool filt = false;
    if (int rc = completions_check(a, dev_image, dev_tokens, token_bytes, n_tokens, dev_offsets, n_rows, filter, h, F, filt)) return rc;
    if (n_rows && (!dev_row_offsets || !dev_ids)) return fail(ACB_EINVAL, "null argument");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_rows == 0) return ACB_OK;
    completions_dispatch<float, kComplEmit>(token_bytes, filt, completions_view(h, dev_image), dev_tokens, n_tokens, dev_offsets, n_rows, F,
                                            nullptr, 0, 0, 0.f, dev_ids, dev_row_offsets, d.sms, static_cast<cudaStream_t>(stream));
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

int acb_completions_mask(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, void *dev_logits, int logits_dtype, int64_t row_stride, int64_t vocab,
                         float value, const acb_pattern_filter *filter, void *stream) {
    ComplHeader h;
    SieveFilter F{};
    bool filt = false;
    if (int rc = completions_check(a, dev_image, dev_tokens, token_bytes, n_tokens, dev_offsets, n_rows, filter, h, F, filt)) return rc;
    if (int rc = completions_logits_check(h, n_rows, dev_logits, logits_dtype, row_stride, vocab)) return rc;
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_rows == 0) return ACB_OK;
    const ComplView V = completions_view(h, dev_image);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (logits_dtype == ACB_LOGITS_F32)
        completions_dispatch<float, kComplMask>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_logits, row_stride,
                                                vocab, value, nullptr, nullptr, d.sms, st);
    else if (logits_dtype == ACB_LOGITS_F16)
        completions_dispatch<__half, kComplMask>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_logits, row_stride,
                                                 vocab, value, nullptr, nullptr, d.sms, st);
    else
        completions_dispatch<__nv_bfloat16, kComplMask>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_logits,
                                                        row_stride, vocab, value, nullptr, nullptr, d.sms, st);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

}  // extern "C"

template <typename T, typename L, bool FILT>
static void completions_bias_launch(const ComplView &V, const void *tokens, uint64_t n_tokens, const int64_t *offsets, int64_t n_rows,
                                    const SieveFilter &F, const float *bias, void *logits, int64_t row_stride, int64_t vocab, int sms,
                                    cudaStream_t st) {
    constexpr int64_t kWarps = kComplThreads / 32;
    int64_t blocks = (n_rows + kWarps - 1) / kWarps;
    if (blocks > 32ll * sms) blocks = 32ll * sms;   // grid-stride beyond that
    completions_bias_kernel<T, L, FILT><<<(unsigned)blocks, kComplThreads, 0, st>>>(
        V, static_cast<const T *>(tokens), n_tokens, offsets, n_rows, F, bias, static_cast<L *>(logits), row_stride, vocab);
}

template <typename L>
static void completions_bias_dispatch(int token_bytes, bool filt, const ComplView &V, const void *tokens, uint64_t n_tokens,
                                      const int64_t *offsets, int64_t n_rows, const SieveFilter &F, const float *bias, void *logits,
                                      int64_t row_stride, int64_t vocab, int sms, cudaStream_t st) {
#define ACB_COMPL_BIAS_LAUNCH(T, FL) \
    completions_bias_launch<T, L, FL>(V, tokens, n_tokens, offsets, n_rows, F, bias, logits, row_stride, vocab, sms, st)
    if (token_bytes == 2) {
        if (filt) ACB_COMPL_BIAS_LAUNCH(uint16_t, true); else ACB_COMPL_BIAS_LAUNCH(uint16_t, false);
    } else if (token_bytes == 4) {
        if (filt) ACB_COMPL_BIAS_LAUNCH(int32_t, true); else ACB_COMPL_BIAS_LAUNCH(int32_t, false);
    } else {
        if (filt) ACB_COMPL_BIAS_LAUNCH(int64_t, true); else ACB_COMPL_BIAS_LAUNCH(int64_t, false);
    }
#undef ACB_COMPL_BIAS_LAUNCH
}

extern "C" {

int acb_completions_bias(const acb_automaton *a, const void *dev_image, const void *dev_tokens, int token_bytes, uint64_t n_tokens,
                         const int64_t *dev_offsets, int64_t n_rows, const float *dev_bias, void *dev_logits, int logits_dtype,
                         int64_t row_stride, int64_t vocab, const acb_pattern_filter *filter, void *stream) {
    ComplHeader h;
    SieveFilter F{};
    bool filt = false;
    if (int rc = completions_check(a, dev_image, dev_tokens, token_bytes, n_tokens, dev_offsets, n_rows, filter, h, F, filt)) return rc;
    if (int rc = completions_logits_check(h, n_rows, dev_logits, logits_dtype, row_stride, vocab)) return rc;
    if (n_rows && !dev_bias) return fail(ACB_EINVAL, "null argument");
    DeviceInfo d;
    if (int rc = device_info(d)) return rc;
    if (n_rows == 0) return ACB_OK;
    const ComplView V = completions_view(h, dev_image);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (logits_dtype == ACB_LOGITS_F32)
        completions_bias_dispatch<float>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_bias, dev_logits, row_stride,
                                         vocab, d.sms, st);
    else if (logits_dtype == ACB_LOGITS_F16)
        completions_bias_dispatch<__half>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_bias, dev_logits, row_stride,
                                          vocab, d.sms, st);
    else
        completions_bias_dispatch<__nv_bfloat16>(token_bytes, filt, V, dev_tokens, n_tokens, dev_offsets, n_rows, F, dev_bias, dev_logits,
                                                 row_stride, vocab, d.sms, st);
    g_launches++;
    CUDA_OK(cudaGetLastError());
    return ACB_OK;
}

}  // extern "C"
