// vocab.cuh -- the vocabulary-mask kernels (acb_vocab_mask): which next ids would complete a string pattern, decided
// over the vocabulary image (vocab.h) for every (row, candidate) pair.
//
// vocab_state_kernel: one warp per history row, grid-stride.  Row i is tokens[a, b) with a, b = offsets[i],
// offsets[i + 1] clamped to [0, n_tokens] (b < a: empty), as for the completions kernels.  The warp reads the ids
// backwards in lane-sized pieces, summing entry lengths (a warp prefix sum) until it holds need = max_pattern_len - 1
// bytes, meets a break (an id outside [0, n_vocab)) or reaches the row start; then lane 0 walks the DFA forward from
// the root over exactly those bytes and writes the row's state.  The ids read are those whose bytes are needed (plus
// any empty entries between them), however long the history.
//
// vocab_mask_kernel: a block holds a tile of kVocabRows rows and strides over the candidate ids, one per thread.  The
// tile's DFA rows (the rows of the states kernel 1 wrote) sit in shared memory, so the first byte of every candidate
// costs one shared load per row, and each id's record is read once per row tile.  Walking candidate t from the row's
// state s: after byte j the walk is in a state of depth d; when d <= j + 1 the string it spells lies inside vocab[t],
// so it is the state the walk from the root reaches after the same j + 1 bytes and the two walks agree from there on.
// Without a filter, t is banned iff some step up to that point enters a match state or tail_hit[t] > j.  Breadth-first
// numbering makes "depth <= 1" the compare s < lvl2, so most ids are decided by one transition.  With a filter a step
// counts only when the entered state's output list holds an admitted pid; tail_hit[t] <= j still proves that no later
// step can hit, and otherwise the walk goes on to byte tail_hit[t] checking the admitted outputs.  A row whose set index
// lies outside [0, n_sets) bans nothing.  Banned pairs get `value` (compl_value rounding); nothing else is written.  A
// thread decides its candidate for all the tile's rows first, into one bit per row, and then stores.
//
// vocab_stop_kernel (acb_vocab_stop): each row's first new id whose bytes end an admitted pattern, by the same
// backwards decode (vocab_tail) and a forward walk over the new ids (below).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "automaton.h"
#include "completions.cuh"
#include "scan_sieve.cuh"
#include "tokens.cuh"
#include "vocab.h"

namespace acb {

constexpr int kVocabThreads = 256;
constexpr int kVocabRows = 16;       // rows per tile of the mask kernel
constexpr int kVocabMaxCols = 256;   // the DFA's widest row
constexpr uint32_t kVocabNoSet = 0xffffffffu;   // a row whose set index lies outside [0, n_sets): it admits nothing

struct VocabView {
    const uint32_t *trans;
    const uint8_t *colmap;
    const uint32_t *match_off, *match_pid, *depth;
    const uint2 *recs;        // VocabRec
    const int32_t *tail;
    const uint8_t *bytes;
    uint32_t n_vocab, n_cols, need, lvl2;
    bool ok;                  // the header's magic matched
};

// the view of an image, read from its header on the device (every thread reads the same few words)
__device__ __forceinline__ VocabView vocab_view(const uint8_t *img) {
    const VocabHeader *h = reinterpret_cast<const VocabHeader *>(img);
    VocabView v;
    v.ok = __ldg(&h->magic) == kVocabMagic;
    v.trans = reinterpret_cast<const uint32_t *>(img + __ldg(&h->off_trans));
    v.colmap = img + __ldg(&h->off_colmap);
    v.match_off = reinterpret_cast<const uint32_t *>(img + __ldg(&h->off_match_off));
    v.match_pid = reinterpret_cast<const uint32_t *>(img + __ldg(&h->off_match_pid));
    v.depth = reinterpret_cast<const uint32_t *>(img + __ldg(&h->off_depth));
    v.recs = reinterpret_cast<const uint2 *>(img + __ldg(&h->off_recs));
    v.tail = reinterpret_cast<const int32_t *>(img + __ldg(&h->off_tail));
    v.bytes = img + __ldg(&h->off_bytes);
    v.n_vocab = __ldg(&h->n_vocab);
    v.n_cols = __ldg(&h->n_cols);
    const uint32_t k = __ldg(&h->max_pat_len);
    v.need = k ? k - 1 : 0;
    v.lvl2 = __ldg(&h->lvl2);
    return v;
}

// The bytes before index `end` of a row whose ids before `end` number `cnt` that can matter: the warp reads the ids
// backwards from end - 1 in lane-sized pieces, summing entry lengths (a warp prefix sum) until it holds need =
// max_pattern_len - 1 bytes, meets a break or has read all `cnt`.  On return every lane holds `start`, the first id a
// forward walk reads, and `skip`, the bytes of that id it skips; start == end when need is 0.
template <typename T>
__device__ __forceinline__ void vocab_tail(const VocabView &V, const T *__restrict__ tokens, uint64_t end, uint64_t cnt, int lane,
                                           uint64_t &start, uint32_t &skip) {
    start = end;
    skip = 0;
    if (!V.need) return;
    uint64_t have = 0;   // bytes of the ids after this piece
    for (uint64_t base = 0;; base += 32) {
        const uint64_t k = base + (uint64_t)lane;   // lane k: the id at end - 1 - k
        const bool valid = k < cnt;
        bool brk = false;
        uint32_t len = 0;
        if (valid) {
            const long long id = token_value(tokens[end - 1 - k]);
            if (id >= 0 && id < (long long)V.n_vocab) len = __ldg(V.recs + id).y;
            else brk = true;
        }
        uint64_t cum = len;   // inclusive prefix sum over the lanes, then the bytes after the piece
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t x = __shfl_up_sync(0xffffffffu, cum, o);
            if (lane >= o) cum += x;
        }
        cum += have;
        const bool reach = valid && !brk && cum >= V.need;
        const unsigned stop = __ballot_sync(0xffffffffu, !valid || brk || reach);
        if (stop) {
            const int f = __ffs(stop) - 1;
            const uint64_t cf = __shfl_sync(0xffffffffu, cum, f);
            const bool rf = (__ballot_sync(0xffffffffu, reach) >> f) & 1u;
            // reached: the id at lane f is the first, minus the bytes beyond `need`; otherwise the walk
            // starts after lane f (a break, or the row start)
            start = end - 1 - (base + (uint64_t)f) + (rf ? 0 : 1);
            skip = rf ? (uint32_t)(cf - V.need) : 0u;
            return;
        }
        have = __shfl_sync(0xffffffffu, cum, 31);
    }
}

// the state the walk from the root reaches over ids [start, end), from byte `skip` of the first (none is a break)
template <typename T>
__device__ __forceinline__ uint32_t vocab_walk(const VocabView &V, const T *__restrict__ tokens, uint64_t start, uint32_t skip,
                                               uint64_t end) {
    uint32_t s = kRoot;
    for (uint64_t i = start; i < end; ++i) {
        const uint2 rc = __ldg(V.recs + token_value(tokens[i]));   // not a break: the scan stopped before any
        for (uint32_t j = i == start ? skip : 0u; j < rc.y; ++j)
            s = __ldg(V.trans + (uint64_t)s * V.n_cols + V.colmap[__ldg(V.bytes + rc.x + j)]) & kStateMask;
    }
    return s;
}

template <typename T>
__global__ void __launch_bounds__(kVocabThreads) vocab_state_kernel(const uint8_t *__restrict__ img, const T *__restrict__ tokens,
                                                                    uint64_t n_tokens, const int64_t *__restrict__ offsets, int64_t n_rows,
                                                                    uint32_t *__restrict__ state) {
    const VocabView V = vocab_view(img);
    if (!V.ok) return;
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (kVocabThreads / 32);
    for (int64_t r = (int64_t)blockIdx.x * (kVocabThreads / 32) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const int64_t o0 = __ldg(offsets + r), o1 = __ldg(offsets + r + 1);
        const uint64_t a = o0 < 0 ? 0 : ((uint64_t)o0 > n_tokens ? n_tokens : (uint64_t)o0);
        uint64_t b = o1 < 0 ? 0 : ((uint64_t)o1 > n_tokens ? n_tokens : (uint64_t)o1);
        if (b < a) b = a;
        uint64_t start;   // the first id the walk reads
        uint32_t skip;    // ... from its byte `skip` on
        vocab_tail(V, tokens, b, b - a, lane, start, skip);
        if (lane == 0) state[r] = vocab_walk(V, tokens, start, skip, b);
    }
}

// does the transition entry e (into state e & kStateMask) count as a hit for the row's set?
template <bool FILT>
__device__ __forceinline__ bool vocab_hit(const VocabView &V, uint32_t e, const uint32_t *row) {
    if (!(e & kMatchFlag)) return false;
    if (!FILT) return true;
    const uint32_t s = e & kStateMask;
    for (uint32_t k = __ldg(V.match_off + s), end = __ldg(V.match_off + s + 1); k < end; ++k)
        if (filter_admits(row, __ldg(V.match_pid + k))) return true;
    return false;
}

// is candidate rc (tail_hit `tail`) banned, e0 being the transition from the row's state over its first byte?
template <bool FILT>
__device__ __forceinline__ bool vocab_banned(const VocabView &V, const uint8_t *colmap, uint32_t e0, uint2 rc, int32_t tail,
                                             const uint32_t *row) {
    if (vocab_hit<FILT>(V, e0, row)) return true;
    uint32_t s = e0 & kStateMask, j = 0;
    if (s >= V.lvl2) {   // depth >= 2 after one byte: walk until the state lies inside the token
        for (;;) {
            if (++j == rc.y) return false;
            const uint32_t e = __ldg(V.trans + (uint64_t)s * V.n_cols + colmap[__ldg(V.bytes + rc.x + j)]);
            if (vocab_hit<FILT>(V, e, row)) return true;
            s = e & kStateMask;
            if (__ldg(V.depth + s) <= j + 1) break;
        }
    }
    // the walk is the root's from byte j on: tail_hit says whether it enters a match state later
    if (tail <= (int32_t)j) return false;
    if (FILT) {   // a later step enters a match state: is any of them admitted?
        while (++j <= (uint32_t)tail) {
            const uint32_t e = __ldg(V.trans + (uint64_t)s * V.n_cols + colmap[__ldg(V.bytes + rc.x + j)]);
            if (vocab_hit<FILT>(V, e, row)) return true;
            s = e & kStateMask;
        }
        return false;
    }
    return true;
}

// row h's set index (filter_row's rule), or kVocabNoSet; the mask ABI keeps n_sets below kVocabNoSet
__device__ __forceinline__ uint32_t vocab_set(const SieveFilter &F, int64_t h) {
    const int64_t s = F.index_bytes == 4 ? (int64_t)__ldg(static_cast<const int32_t *>(F.index) + h)
                                         : (int64_t)__ldg(static_cast<const long long *>(F.index) + h);
    return s >= 0 && (uint64_t)s < F.n_sets ? (uint32_t)s : kVocabNoSet;
}

template <typename L, bool FILT>
__global__ void __launch_bounds__(kVocabThreads) vocab_mask_kernel(const uint8_t *__restrict__ img, const uint32_t *__restrict__ state,
                                                                   int64_t n_rows, SieveFilter F, L *__restrict__ logits, int64_t row_stride,
                                                                   int64_t vocab, float value) {
    __shared__ uint32_t rows[kVocabRows * kVocabMaxCols];   // the tile's DFA rows
    __shared__ uint32_t sets[kVocabRows];                   // the tile's set indexes
    __shared__ uint8_t colmap[256];
    const VocabView V = vocab_view(img);
    if (!V.ok) return;
    const L fill = compl_value<L>(value);
    const int64_t limit = vocab < (int64_t)V.n_vocab ? vocab : (int64_t)V.n_vocab;   // the candidates
    if ((int64_t)blockIdx.x * kVocabThreads >= limit) return;   // no candidate for this block (V > n_vocab)
    for (int k = threadIdx.x; k < 256; k += kVocabThreads) colmap[k] = __ldg(V.colmap + k);
    const int64_t tiles = (n_rows + kVocabRows - 1) / kVocabRows;
    for (int64_t tile = blockIdx.y; tile < tiles; tile += gridDim.y) {
        const int64_t r0 = tile * kVocabRows;
        const int nr = (int)min((int64_t)kVocabRows, n_rows - r0);
        __syncthreads();   // the previous tile's rows are no longer read
        for (int k = threadIdx.x; k < nr * (int)V.n_cols; k += kVocabThreads) {
            const int r = k / (int)V.n_cols, c = k - r * (int)V.n_cols;
            rows[r * kVocabMaxCols + c] = __ldg(V.trans + (uint64_t)__ldg(state + r0 + r) * V.n_cols + c);
        }
        if (FILT && threadIdx.x < nr) sets[threadIdx.x] = vocab_set(F, r0 + threadIdx.x);
        __syncthreads();
        for (int64_t t = (int64_t)blockIdx.x * kVocabThreads + threadIdx.x; t < limit; t += (int64_t)gridDim.x * kVocabThreads) {
            const uint2 rc = __ldg(V.recs + t);
            if (rc.y == 0) continue;   // an empty entry completes nothing
            const int32_t tail = __ldg(V.tail + t);
            const uint32_t c0 = colmap[__ldg(V.bytes + rc.x)];
            uint32_t hit = 0;   // bit r: t is banned for row r0 + r
            for (int r = 0; r < nr; ++r) {
                const uint32_t *set = nullptr;
                if (FILT) {
                    if (sets[r] == kVocabNoSet) continue;
                    set = F.bits + (uint64_t)sets[r] * F.words;
                }
                if (vocab_banned<FILT>(V, colmap, rows[r * kVocabMaxCols + c0], rc, tail, set)) hit |= 1u << r;
            }
            // The stores come after the walks, and each store's row comes from this thread's own bits.  A version that
            // stored inside the row loop was miscompiled by ptxas (CUDA 12.9) in its 16-bit filtered instances: the
            // row of the store address was taken from a uniform register (R2UR of the loop counter) while the lanes of
            // a warp were at different rows of their walks, so some bans went to another row of the tile (DESIGN §4.18).
            for (L *col = logits + t; hit; hit &= hit - 1) col[(r0 + (__ffs(hit) - 1)) * row_stride] = fill;
        }
    }
}

// vocab_stop_kernel: one warp per row, grid-stride.  Row i is clamped as for vocab_state_kernel; its last
// min(max(new_i, 0), b - a) ids are new (new_i = news[i], or n_new when news is null), the first of them at f.  The warp
// decodes backwards from f (vocab_tail), then lane 0 walks the DFA from the root over those bytes and on over the new
// ids' bytes: a break resets the walk to the root, an empty entry adds nothing.  The first entered state with an
// admitted output ends the walk: the first admitted pid of its output list (own patterns, then suffixes, longest first,
// ties by ascending pid) is the row's stop, the occurrence with the earliest last byte inside a new id, the longest of
// those.  out[4i .. 4i + 3] = (pid, token index from a, bytes of that id up to the match's last byte, pattern length),
// or -1 four times.  The walk over the new ids is serial: meant for a decoding step's few ids, not a whole document.
// The walk from state s over ids [i, b): a break resets it to the root, an empty entry adds nothing.  True when it
// enters a state with an admitted output; then i, j and s are that id, its byte and the state.
template <typename T, bool FILT>
__device__ __forceinline__ bool vocab_stop_walk(const VocabView &V, const T *__restrict__ tokens, uint32_t s0, uint64_t b,
                                                const uint32_t *set, uint64_t &i, uint32_t &j, uint32_t &s) {
    s = s0;
    for (; i < b; ++i) {
        const long long id = token_value(tokens[i]);
        if (id < 0 || id >= (long long)V.n_vocab) {   // a break: no occurrence spans it
            s = kRoot;
            continue;
        }
        const uint2 rc = __ldg(V.recs + id);
        for (j = 0; j < rc.y; ++j) {
            const uint32_t e = __ldg(V.trans + (uint64_t)s * V.n_cols + V.colmap[__ldg(V.bytes + rc.x + j)]);
            s = e & kStateMask;
            if (vocab_hit<FILT>(V, e, set)) return true;
        }
    }
    return false;
}

template <typename T, bool FILT>
__global__ void __launch_bounds__(kVocabThreads) vocab_stop_kernel(const uint8_t *__restrict__ img, const T *__restrict__ tokens,
                                                                   uint64_t n_tokens, const int64_t *__restrict__ offsets, int64_t n_rows,
                                                                   int64_t n_new, const int64_t *__restrict__ news, SieveFilter F,
                                                                   int64_t *__restrict__ out) {
    const VocabView V = vocab_view(img);
    if (!V.ok) return;
    const uint8_t *dfa = img + __ldg(&reinterpret_cast<const VocabHeader *>(img)->off_dfa);
    const uint32_t *pat_len = reinterpret_cast<const uint32_t *>(dfa + __ldg(&reinterpret_cast<const ImageHeader *>(dfa)->off_pat_len));
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (kVocabThreads / 32);
    for (int64_t r = (int64_t)blockIdx.x * (kVocabThreads / 32) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const int64_t o0 = __ldg(offsets + r), o1 = __ldg(offsets + r + 1);
        const uint64_t a = o0 < 0 ? 0 : ((uint64_t)o0 > n_tokens ? n_tokens : (uint64_t)o0);
        uint64_t b = o1 < 0 ? 0 : ((uint64_t)o1 > n_tokens ? n_tokens : (uint64_t)o1);
        if (b < a) b = a;
        const int64_t nw = news ? __ldg(news + r) : n_new;
        const uint64_t f = b - (nw <= 0 ? 0 : ((uint64_t)nw > b - a ? b - a : (uint64_t)nw));   // the first new id
        uint64_t start;
        uint32_t skip;
        vocab_tail(V, tokens, f, f - a, lane, start, skip);
        if (lane == 0) {
            const uint32_t *set = FILT ? filter_row(F, r) : nullptr;
            uint64_t i = f;   // the id, and its byte j, where the walk enters a state with an admitted output
            uint32_t j = 0, s = kRoot;
            const bool hit = (!FILT || set) && vocab_stop_walk<T, FILT>(V, tokens, vocab_walk(V, tokens, start, skip, f), b, set, i, j, s);
            int64_t *o = out + 4 * r;
            if (hit) {
                uint32_t k = __ldg(V.match_off + s);   // the first admitted pid of s's output list
                if (FILT)
                    while (!filter_admits(set, __ldg(V.match_pid + k))) ++k;
                const uint32_t pid = __ldg(V.match_pid + k);
                o[0] = pid;
                o[1] = (int64_t)(i - a);
                o[2] = (int64_t)j + 1;
                o[3] = __ldg(pat_len + pid);
            } else {
                o[0] = o[1] = o[2] = o[3] = -1;
            }
        }
    }
}

}  // namespace acb
