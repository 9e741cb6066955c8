// completions.cuh -- the completing-token kernels (acb_completions_count / _emit / _mask, and _bias in its own kernel
// below): one warp per history row, grid-stride over the rows, walking the completions image (completions.h) from the
// root backwards over the row's last ids.
//
// Row i's history is tokens[a, b) with a, b = offsets[i], offsets[i + 1] clamped to [0, n_tokens] (b < a: empty),
// so no offset is ever trusted and nothing is read outside `tokens`.  Only its last min(b - a, depth) ids are read,
// in lane-sized pieces: the work per row does not grow with the history.  An id outside [0, 2^21) equals no pattern
// token, so the walk stops there.  With a filter, an entry counts only when its pid is admitted by the row's set
// (SieveFilter, scan_sieve.cuh; an index outside [0, n_sets) admits nothing).
//
//   MASK   logits[row * row_stride + token] = value for every admitted entry on the path.  A token may be written
//          twice (from two pids or two depths): the same value, harmless.
//   COUNT  counts[row] = the number of DISTINCT admitted tokens on the path.
//   EMIT   those tokens, written from ids[row_offsets[row]]; ascending within a node, nodes root first.
// COUNT and EMIT report an entry only when it is its token's first admitted occurrence: no admitted entry with the
// same token earlier in its node (entries sort by (token, pid)) nor at any shallower node of the path -- the path's
// shallower nodes are the node's ancestors, found through elink.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "completions.h"
#include "scan_sieve.cuh"
#include "tokens.cuh"

namespace acb {

enum ComplMode { kComplMask = 0, kComplCount = 1, kComplEmit = 2 };
constexpr int kComplThreads = 256;

struct ComplView {
    const ComplNode *nodes;
    const uint32_t *kid_tok;
    const ComplEntry *entries;
    uint32_t depth;
};

template <typename L>
__device__ __forceinline__ L compl_value(float v);
template <>
__device__ __forceinline__ float compl_value<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half compl_value<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 compl_value<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <bool FILT>
__device__ __forceinline__ bool compl_admits(const uint32_t *row, uint32_t pid) {
    return !FILT || filter_admits(row, pid);
}

// is entry e (token t) of node v the first admitted occurrence of t on the path that ends at v?
template <bool FILT>
__device__ bool compl_first(const ComplView &V, const uint32_t *row, const ComplNode &nd, uint32_t e, uint32_t t) {
    for (uint32_t k = e; k-- > nd.first_entry;) {
        const ComplEntry x = V.entries[k];
        if (x.token != t) break;
        if (compl_admits<FILT>(row, x.pid)) return false;
    }
    for (uint32_t u = nd.elink; u != kComplNone;) {
        const ComplNode an = V.nodes[u];
        uint32_t lo = an.first_entry, hi = an.first_entry + an.n_entries;   // lower bound of t
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (V.entries[mid].token < t) lo = mid + 1;
            else hi = mid;
        }
        for (; lo < an.first_entry + an.n_entries; ++lo) {
            const ComplEntry x = V.entries[lo];
            if (x.token != t) break;
            if (compl_admits<FILT>(row, x.pid)) return false;
        }
        u = an.elink;
    }
    return true;
}

// the child of nd that prepends token t, or kComplNone: a 32-ary warp search of the sorted child tokens (the root
// can have tens of thousands of children), then one compare per lane
__device__ __forceinline__ uint32_t compl_child(const ComplView &V, const ComplNode &nd, uint32_t t, int lane) {
    uint32_t lo = nd.first_kid, n = nd.n_kids;
    while (n > 32) {
        const uint32_t step = (n + 31) / 32;
        const uint32_t at = (uint32_t)lane * step;
        const bool le = at < n && __ldg(V.kid_tok + lo + at) <= t;
        const unsigned bal = __ballot_sync(0xffffffffu, le);
        if (!bal) return kComplNone;
        const uint32_t c = 31u - __clz(bal);   // the last sample <= t (the samples ascend)
        lo += c * step;
        n = min(step, n - c * step);
    }
    const bool eq = (uint32_t)lane < n && __ldg(V.kid_tok + lo + lane) == t;
    const unsigned bal = __ballot_sync(0xffffffffu, eq);
    return bal ? lo + (uint32_t)(__ffs(bal) - 1) : kComplNone;
}

template <typename T, typename L, int MODE, bool FILT>
__global__ void __launch_bounds__(kComplThreads) completions_kernel(ComplView V, const T *__restrict__ tokens, uint64_t n_tokens,
                                                                    const int64_t *__restrict__ offsets, int64_t n_rows, SieveFilter F,
                                                                    L *__restrict__ logits, int64_t row_stride, int64_t vocab, float value,
                                                                    int64_t *__restrict__ out, const int64_t *__restrict__ out_offsets) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (kComplThreads / 32);
    const L fill = compl_value<L>(value);
    for (int64_t r = (int64_t)blockIdx.x * (kComplThreads / 32) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const int64_t o0 = __ldg(offsets + r), o1 = __ldg(offsets + r + 1);
        const uint64_t a = o0 < 0 ? 0 : ((uint64_t)o0 > n_tokens ? n_tokens : (uint64_t)o0);
        uint64_t b = o1 < 0 ? 0 : ((uint64_t)o1 > n_tokens ? n_tokens : (uint64_t)o1);
        if (b < a) b = a;
        const uint32_t m = (uint32_t)min((uint64_t)V.depth, b - a);   // ids the walk may read
        const uint32_t *row = FILT ? filter_row(F, r) : nullptr;
        int64_t found = 0;   // COUNT / EMIT: distinct tokens so far (every lane)
        int64_t base = 0;
        if (MODE == kComplEmit) base = __ldg(out_offsets + r);
        if (!FILT || row != nullptr) {
            uint32_t v = 0;
            long long piece = 0;   // lane k: the id at b - 1 - (d & ~31) - k
            for (uint32_t d = 0;; ++d) {
                const ComplNode nd = V.nodes[v];
                for (uint32_t k0 = 0; k0 < nd.n_entries; k0 += 32) {
                    const uint32_t e = nd.first_entry + k0 + lane;
                    bool hit = false;
                    uint32_t t = 0;
                    if (k0 + lane < nd.n_entries) {
                        const ComplEntry x = V.entries[e];
                        t = x.token;
                        hit = compl_admits<FILT>(row, x.pid);
                        if (MODE == kComplMask) {
                            if (hit && (int64_t)t < vocab) logits[r * row_stride + t] = fill;
                        } else if (hit) {
                            hit = compl_first<FILT>(V, row, nd, e, t);
                        }
                    }
                    if (MODE != kComplMask) {
                        const unsigned bal = __ballot_sync(0xffffffffu, hit);
                        if (MODE == kComplEmit && hit) out[base + found + __popc(bal & ((1u << lane) - 1u))] = t;
                        found += __popc(bal);
                    }
                }
                if (d == m) break;
                if ((d & 31u) == 0) {
                    const uint32_t k = d + (uint32_t)lane;
                    piece = k < m ? token_value(tokens[b - 1 - k]) : 0;
                }
                const long long id = __shfl_sync(0xffffffffu, piece, (int)(d & 31u));
                if (!token_ok(id)) break;   // equals no pattern token
                v = compl_child(V, nd, (uint32_t)id, lane);
                if (v == kComplNone) break;
            }
        }
        if (MODE == kComplCount && lane == 0) out[r] = found;
    }
}

template <typename L>
__device__ __forceinline__ float compl_float(L x);
template <>
__device__ __forceinline__ float compl_float<float>(float x) { return x; }
template <>
__device__ __forceinline__ float compl_float<__half>(__half x) { return __half2float(x); }
template <>
__device__ __forceinline__ float compl_float<__nv_bfloat16>(__nv_bfloat16 x) { return __bfloat162float(x); }

// adds to s (has: s holds a term already) bias[pid] of every admitted entry with token t from entries[k] on, in pid
// order; the sum starts from its first term, so a lone -0.0 stays -0.0
template <bool FILT>
__device__ __forceinline__ void compl_bias_run(const ComplView &V, const uint32_t *row, const float *bias, uint32_t k, uint32_t end,
                                               uint32_t t, float &s, bool &has) {
    for (; k < end; ++k) {
        const ComplEntry x = V.entries[k];
        if (x.token != t) break;
        if (!compl_admits<FILT>(row, x.pid)) continue;
        const float b = __ldg(bias + x.pid);
        s = has ? __fadd_rn(s, b) : b;
        has = true;
    }
}

// The bias mode (acb_completions_bias), a sibling of completions_kernel: logits[row * row_stride + t] += the sum of
// bias[pid] over the admitted pids that t completes, longest pattern first, ties by ascending pid, summed in float32
// from the first term and rounded to L once.  The warp walks to the deepest path node v_end touching no entries, then
// visits the path's nodes with entries deepest first (v_end or its elink, then elink): that is the sum's order, as
// deeper nodes spell longer p[:-1] and a node's entries sort by (token, pid).  The lane that holds t's first admitted
// occurrence on the path (compl_first, the shallowest) owns t: it sums the admitted entries of t at every chain node
// from v_end down to its own, one lower-bound search per node, then its own node's run from its entry on (compl_first
// says no ancestor holds an admitted t), and makes the one read-modify-write of the element.  No atomics, so the
// result is reproducible bit for bit.
template <typename T, typename L, bool FILT>
__global__ void __launch_bounds__(kComplThreads) completions_bias_kernel(ComplView V, const T *__restrict__ tokens, uint64_t n_tokens,
                                                                         const int64_t *__restrict__ offsets, int64_t n_rows, SieveFilter F,
                                                                         const float *__restrict__ bias, L *__restrict__ logits,
                                                                         int64_t row_stride, int64_t vocab) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (kComplThreads / 32);
    for (int64_t r = (int64_t)blockIdx.x * (kComplThreads / 32) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const int64_t o0 = __ldg(offsets + r), o1 = __ldg(offsets + r + 1);
        const uint64_t a = o0 < 0 ? 0 : ((uint64_t)o0 > n_tokens ? n_tokens : (uint64_t)o0);
        uint64_t b = o1 < 0 ? 0 : ((uint64_t)o1 > n_tokens ? n_tokens : (uint64_t)o1);
        if (b < a) b = a;
        const uint32_t m = (uint32_t)min((uint64_t)V.depth, b - a);   // ids the walk may read
        const uint32_t *row = FILT ? filter_row(F, r) : nullptr;
        if (FILT && row == nullptr) continue;   // the row's set index admits nothing
        uint32_t v = 0;
        long long piece = 0;   // lane k: the id at b - 1 - (d & ~31) - k
        for (uint32_t d = 0; d < m; ++d) {
            if ((d & 31u) == 0) {
                const uint32_t k = d + (uint32_t)lane;
                piece = k < m ? token_value(tokens[b - 1 - k]) : 0;
            }
            const long long id = __shfl_sync(0xffffffffu, piece, (int)(d & 31u));
            if (!token_ok(id)) break;   // equals no pattern token
            const uint32_t c = compl_child(V, V.nodes[v], (uint32_t)id, lane);
            if (c == kComplNone) break;
            v = c;
        }
        const ComplNode end = V.nodes[v];
        const uint32_t top = end.n_entries ? v : end.elink;   // the deepest path node with entries
        for (uint32_t u = top; u != kComplNone;) {
            const ComplNode nd = V.nodes[u];
            for (uint32_t k0 = lane; k0 < nd.n_entries; k0 += 32) {
                const uint32_t e = nd.first_entry + k0;
                const ComplEntry x = V.entries[e];
                const uint32_t t = x.token;
                if ((int64_t)t >= vocab || !compl_admits<FILT>(row, x.pid) || !compl_first<FILT>(V, row, nd, e, t)) continue;
                float s = 0.f;
                bool has = false;
                for (uint32_t w = top; w != u;) {   // the deeper chain nodes, deepest first
                    const ComplNode cn = V.nodes[w];
                    const uint32_t hi0 = cn.first_entry + cn.n_entries;
                    uint32_t lo = cn.first_entry, hi = hi0;   // lower bound of t
                    while (lo < hi) {
                        const uint32_t mid = (lo + hi) >> 1;
                        if (V.entries[mid].token < t) lo = mid + 1;
                        else hi = mid;
                    }
                    compl_bias_run<FILT>(V, row, bias, lo, hi0, t, s, has);
                    w = cn.elink;
                }
                compl_bias_run<FILT>(V, row, bias, e, nd.first_entry + nd.n_entries, t, s, has);
                L *p = logits + r * row_stride + t;
                *p = compl_value<L>(__fadd_rn(compl_float<L>(*p), s));
            }
            u = nd.elink;
        }
    }
}

}  // namespace acb
