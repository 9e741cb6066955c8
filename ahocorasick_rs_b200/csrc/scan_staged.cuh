// scan_staged.cuh -- the hot kernel: one lane per SEGMENT of the byte stream,
// hot table rows in shared memory, bytes staged through shared memory with
// cp.async.
//
// Layout per CTA (dynamic shared memory):
//   [ hot table : (H + 1) rows x n_cols u16 ]  rows 0..H-1 are the H hottest
//        states of the hot image (automaton.h: HotHeader; ranked by sampled
//        visit counts).  An entry is the BYTE OFFSET of the next state's row
//        inside this table when that state is hot and is neither a match state
//        nor the dead state, else the offset of row H, the TRAP row, which maps
//        everything to itself.  Brought in with one TMA bulk copy
//        (cp.async.bulk + mbarrier) when the whole hot image fits; the CTA then
//        adds the table's own shared-memory address to every entry, so an entry
//        IS the 32-bit shared address of the next row: one multiply-add
//        (row + 2 * column, an IMAD on the otherwise idle FMA pipe; an IDP.4A
//        straight from the data word for the byte-indexed table) forms the next
//        load address, with nothing else on the dependent chain.  A lane that left the hot set stays trapped and
//        ONE compare per 64 bytes detects it; only the group something happened
//        in is redone, through the exact scanner.  (Addresses must fit 16 bits:
//        the table lives in the first 64 KB of shared memory.)
//   [ column map : 256 B ]  (kColClass only)
//   [ mbarrier, stream bounds; each warp's current task ]
//   [ hot2full : (H + 1) x u32 ]  hot row -> automaton state, for the segment
//        summaries and the hand-over to the exact scanner
//   [ metadata : per warp 32 V x (first 16-byte unit, number of chunks, guessed start
//        state, how the first chunk is fetched) ]  the first two are read by the copy
//        issue; the guess waits there for the segment summary
//   [ staging : per warp, 2 buffers x 32 V rows x 64 B ]  lane l's 64-byte
//        chunk is row l, with its four 16-byte units XOR-swizzled by
//        (l >> 1) & 3: the per-lane LDS.128 reads of a quarter warp hit 8
//        different bank groups (conflict free), and a warp-wide cp.async
//        instruction (8 rows) fills four whole 128-byte lines of shared
//        memory.  (An 80-byte pitch without a swizzle reads just as well, but
//        every copy instruction then straddles 12-14 lines instead of 8, the
//        floor.)
//   V = segments per lane (template parameter): 1, or 2 whose chains interleave.
//
// All shared-memory traffic of the scan loop goes through explicit 32-bit
// shared addresses (inline PTX): the swizzle is an XOR on the address, and the
// table loads must not pick up a base-address add on the dependent chain.
//
// Work decomposition (scan_core.cuh: SegPlan).  The stream is cut into
// fixed-size segments; a lane scans one segment, walking through whatever
// haystack boundaries fall inside it (each haystack start resets the scanner to
// the root, exactly).  A segment that begins inside a haystack begins with a
// speculated state: the lane first scans `warm` bytes before the segment from
// the root, silently, and takes the state it arrives with.  It records that
// state and its end state in the segment summary (SegOut); repair.cuh verifies the chain and redoes
// the few places where the guess was wrong.  Lanes of a warp take segments
// `lane_stride` apart, which for a batch of equal-length haystacks puts all 32
// lanes at the same offset of 32 different haystacks (same text -> same table
// row -> shared-memory broadcasts instead of bank conflicts).
//
// Each lane reads its bytes in 64-byte chunks of the ABSOLUTE address grid,
// so every cp.async is 16-byte aligned and a warp-wide copy instruction
// touches 8 x 64 contiguous bytes.  Chunk k+1 is in flight while chunk k is
// scanned.  The copies ask the L2 for whole 128-byte lines: a lane's rows are
// 4 KiB apart, and fetching two chunks of a row per DRAM access instead of one
// is what keeps the warps fed.  The copy of the chunk that completes a line
// marks it evict_first, so the spent stream leaves the L2 first (DESIGN.md §6;
// a third staging buffer and L2 prefetches of a lane's later bytes were slower).
// The warm-up bytes are the exception: they end the neighbouring segment's last
// line, so the first chunk of such a segment copies only the 16-byte units that
// hold them, sector by sector, and leaves the line to the lane that scans it.
//
// Where a lane's state lives.  The chunk loop keeps position, table row, piece
// end and a few predicates per segment in registers.  The exact scanner's state
// and the segment bookkeeping (PieceCtx, LaneSeg: 28 words in local memory)
// exist only for a lane that has needed the exact scanner: it builds them then
// (seg_setup + build_cold) from the task number, its lane and the guess in its
// metadata row.  A lane that stays on the fast path -- all but about 2 % of
// config 2's -- writes its summary from registers and shared memory and never
// touches local memory.
#pragma once
#include <type_traits>

#include "scan_core.cuh"

namespace acb {

#ifndef ACB_MAX_WARPS
#define ACB_MAX_WARPS 32
#endif
constexpr int kMaxWarps = ACB_MAX_WARPS;  // per CTA (one CTA per SM): 32 -> 64 registers per thread, 28 -> 72, 24 -> 80
#ifndef ACB_MAX_WARPS2
#define ACB_MAX_WARPS2 22
#endif
constexpr int kMaxWarps2 = ACB_MAX_WARPS2;  // two segments per lane: twice the staging per warp, up to 88 registers
constexpr int kChunk = 64;                // bytes per lane per stage
constexpr int kRow = kChunk;              // a lane's row in the staging buffer; its 16-byte units are swizzled by (lane >> 1) & 3
constexpr int kStageBytes = 32 * kRow;    // per warp per buffer and per segment of a lane
constexpr int kStageOffset = 256 + 128 + 4 * kMaxWarps;  // column map, mbarrier slot + stream bounds, each warp's current task, after the hot table
constexpr int kMetaRow = 16;              // per segment of a lane: first 16-byte unit and chunk count (read by the copy issue), the guessed
                                          // state at the segment start, how the first chunk is fetched (SegSetup::first_fetch)
constexpr int kMetaBytes = 32 * kMetaRow; // per warp and per segment of a lane

struct FastTab {
    uint32_t cmap;  // shared address of the byte -> column map (kColClass)
    uint32_t lo, maxc;
};

// ---- shared memory by 32-bit shared address ----
// Table loads: the table never changes after the prologue, so the load is a pure function of its
// address (not volatile: the compiler may schedule it freely).
__device__ __forceinline__ uint32_t lds_tab(uint32_t addr) {
    uint32_t v;
    asm("ld.shared.u16 %0, [%1];\n" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_tab_u8(uint32_t addr) {
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];\n" : "=r"(v) : "r"(addr));
    return v;
}
// Staged bytes and copy metadata: volatile, the same address holds different data from one chunk to the next.
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];\n" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(addr));  // (only used on tables that never change after the prologue)
    return v;
}
__device__ __forceinline__ uint32_t lds32v(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, uint2 v) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};\n" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}
// a lane's staged row: `row` is the address of its 16-byte unit 0; unit j and byte p of the swizzled row
__device__ __forceinline__ uint32_t row_unit(uint32_t row, uint32_t j) { return row ^ (j << 4); }
__device__ __forceinline__ uint32_t row_byte(uint32_t row, uint32_t p) { return (row ^ (p & 0x30u)) + (p & 15u); }

constexpr int kColAscii = 2;  // hot table indexed by the raw byte (128 entries per row); bytes >= 128 clamp to 127

// one transition: s is the shared address of the current row, the result that of the next
template <int COLMODE, bool CLAMP = true>
__device__ __forceinline__ uint32_t fstep(uint32_t s, uint32_t b, const FastTab &f) {
    uint32_t col;
    if (COLMODE == kColRange)
        col = min(b - f.lo, f.maxc);
    else if (COLMODE == kColClass)
        col = lds_tab_u8(f.cmap + b);
    else
        col = CLAMP ? min(b, 127u) : b;
    // row + 2 * column as an IMAD: the kernel is bound by the ALU pipe (half rate; the byte extract and the
    // column clamp live there), the multiply-add pipe is idle
    uint32_t addr;
    asm("mad.lo.u32 %0, %1, 2, %2;\n" : "=r"(addr) : "r"(col), "r"(s));
    return lds_tab(addr);
}

// byte-indexed table: row + 2 * byte k of w in ONE instruction (IDP4A: w . (2 << 8k) + row), no byte extract
template <uint32_t K>
__device__ __forceinline__ uint32_t fstep_dp(uint32_t s, uint32_t w) {
    uint32_t addr;
    asm("dp4a.u32.u32 %0, %1, %2, %3;\n" : "=r"(addr) : "r"(w), "r"(2u << (8 * K)), "r"(s));
    return lds_tab(addr);
}
// bytes >= 0x80 of a word -> 0x7f (the byte-indexed table's "any other byte" column)
__device__ __forceinline__ uint32_t clamp7f(uint32_t w) {
    const uint32_t hi = w & 0x80808080u;
    return (w | (hi - (hi >> 7))) & ~hi;
}

template <int COLMODE, bool CLAMP = true>
__device__ __forceinline__ uint32_t fstep4(uint32_t s, uint32_t w, const FastTab &f) {
    if (COLMODE == kColAscii && !CLAMP) {
        // the caller has clamped the word's bytes to 0..127 already
        s = fstep_dp<0>(s, w);
        s = fstep_dp<1>(s, w);
        s = fstep_dp<2>(s, w);
        return fstep_dp<3>(s, w);
    }
    s = fstep<COLMODE, CLAMP>(s, __byte_perm(w, 0, 0x4440), f);
    s = fstep<COLMODE, CLAMP>(s, __byte_perm(w, 0, 0x4441), f);
    s = fstep<COLMODE, CLAMP>(s, __byte_perm(w, 0, 0x4442), f);
    s = fstep<COLMODE, CLAMP>(s, __byte_perm(w, 0, 0x4443), f);
    return s;
}

// continuation bytes (10xxxxxx) in a word
__device__ __forceinline__ uint32_t cont_bytes(uint32_t w) { return __popc(w & ~(w << 1) & 0x80808080u); }

// .L2::128B: the L2 fetches the whole 128-byte line, not just the 64 bytes a lane's chunk needs, so the next chunk of
// the row is usually in L2 by the time it is copied (DESIGN.md §6).  src must be a valid address even when
// src_bytes is 0.
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16, %2;\n" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
// The same with an evict_first L2 policy, for the copy of the chunk that completes its 128-byte line: that line is
// spent, so the L2 gives it up before anything else.  (evict_first on every copy is much slower: the first half's
// copy would evict the line before the second half is read.  DESIGN.md §6.)
__device__ __forceinline__ void cp_async16_last(uint32_t dst_smem, const void *src, uint32_t src_bytes) {
    asm volatile(
        "{\n"
        ".reg .b64 pol;\n"
        "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n"
        "cp.async.cg.shared.global.L2::cache_hint.L2::128B [%0], [%1], 16, %2, pol;\n"
        "}\n" ::"r"(dst_smem), "l"(src), "r"(src_bytes)
        : "memory");
}
// A plain 16-byte copy, no prefetch size and no policy: DRAM supplies one 32-byte sector.  For the warm-up bytes before a
// segment: the rest of their 128-byte line belongs to the neighbouring segment, whose lane reads it at another time.
__device__ __forceinline__ void cp_async16_sector(uint32_t dst_smem, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// ---- TMA bulk copy (global -> shared) completing on an mbarrier ----
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

// Views into the hot image (global memory).
struct DevHot {
    const uint16_t *table;
    const uint32_t *hot2full;
    const uint16_t *full2hot;
    uint32_t n_rows;
    const uint16_t *table128;  // kColAscii
    uint32_t n_rows128;
};

// What a lane knows about its segment besides the scanner state (kept out of
// the hot loop's registers: only touched at piece boundaries).
enum PieceKind : uint32_t { kPieceWarm = 0, kPieceHead = 1, kPieceNormal = 2 };
struct LaneSeg {
    int64_t org;         // stream position of c.base
    int64_t seg;         // segment index
    uint32_t lo_rel, hi_rel;  // the segment, relative to org
    uint32_t h;          // current haystack
    uint32_t kind;
    uint32_t spec_state, head_count;
    uint32_t done;
    uint32_t far;        // code points: the segment starts more than kContSpan segments into its haystack
};

// Where a lane's segment lies and how its scan starts: a pure function of the task, the lane and the batch.  The task
// start keeps what the chunk loop needs in registers; the rest is derived again when a lane first needs the exact
// scanner (build_cold), so a lane that never does stores none of it.
struct SegSetup {
    int64_t seg, org, hs;     // segment index; stream position of relative position 0 (a 64-byte aligned address); start of the haystack
    uint32_t h;               // the haystack the scan starts in
    uint32_t lo_rel, hi_rel;  // the segment, relative to org
    uint32_t at, limit;       // where the scan starts (the warm-up bytes before lo_rel, if any), and the end of the haystack
    uint32_t off16;           // 16-byte unit of org on the copy grid
    uint32_t first_fetch;     // a warm-up: kWarmFetch | first 16-byte unit of chunk 0 that the scan reads; else 0
    bool live, outside;       // has bytes to scan; lies in the plan but outside the stream (an empty summary is due)
    bool cont;                // begins inside a haystack: `warm` bytes before it are scanned silently first
};
constexpr uint32_t kWarmFetch = 0x80000000u;

template <int V>
__device__ __forceinline__ int64_t seg_of_lane(const SegPlan &P, unsigned int task, uint32_t vlane) {
    const uint32_t q = P.lane_stride;
    return (int64_t)(((uint64_t)(task / q) * (32u * V) + vlane) * q + task % q);
}

template <int V>
__device__ __forceinline__ SegSetup seg_setup(const SegPlan &P, const Batch &B, int64_t stream_lo, int64_t stream_hi, uintptr_t gbase,
                                              unsigned int task, uint32_t vlane) {
    SegSetup u;
    u.seg = seg_of_lane<V>(P, task, vlane);
    u.org = u.hs = 0;
    u.h = u.lo_rel = u.hi_rel = u.at = u.limit = u.off16 = u.first_fetch = 0;
    u.cont = false;
    const int64_t glo = P.origin + u.seg * (int64_t)P.seg_bytes;
    const int64_t lo = max(glo, stream_lo), hi = min(glo + (int64_t)P.seg_bytes, stream_hi);
    u.live = u.seg < P.n_segments && lo < hi;
    u.outside = u.seg < P.n_segments && lo >= hi;  // (the plan is sized from the buffer length)
    if (u.live) {
        // the haystack containing lo: try the position an equal-length batch would put it at, else search
        // (32-bit arithmetic: a buffer is shorter than 4 GiB)
        int64_t h = P.avg_len ? (int64_t)((uint32_t)(lo - stream_lo) / (uint32_t)P.avg_len) : 0;
        if (h >= B.n_haystacks) h = B.n_haystacks - 1;
        int64_t hs = __ldg(B.offsets + h), he = __ldg(B.offsets + h + 1);
        if (!(hs <= lo && lo < he)) {
            h = find_haystack(B, lo);
            hs = __ldg(B.offsets + h);
            he = __ldg(B.offsets + h + 1);
        }
        u.cont = hs < lo;
        const int64_t w = u.cont ? max(hs, lo - (int64_t)P.warm) : lo;
        const uintptr_t pw = reinterpret_cast<uintptr_t>(B.bytes + w);
        const uintptr_t a0 = pw & ~uintptr_t(kChunk - 1);
        u.org = w - (int64_t)(pw - a0);
        u.hs = hs;
        u.h = (uint32_t)h;
        u.lo_rel = (uint32_t)(lo - u.org);
        u.hi_rel = (uint32_t)(hi - u.org);
        u.at = (uint32_t)(w - u.org);
        u.limit = (uint32_t)(he - u.org);
        u.off16 = (uint32_t)((a0 - gbase) >> 4);
        u.first_fetch = u.cont ? kWarmFetch | (u.at >> 4) : 0u;
    }
    return u;
}

// The exact scanner's state and the segment bookkeeping of a lane that has only run the fast path so far: nothing
// reported, nothing pending.  `warm`: still in the warm-up; else `spec` is the state guessed at the segment start
// (kNoState when the segment starts its haystack).  c.at, c.state and the code-point counters are the caller's.
template <bool CP>
__device__ __forceinline__ void build_cold(PieceCtx &c, LaneSeg &L, const SegSetup &u, const SegPlan &P, const Batch &B, bool warm,
                                           uint32_t spec) {
    L.org = u.org;
    L.seg = u.seg;
    L.lo_rel = u.lo_rel;
    L.hi_rel = u.hi_rel;
    L.h = u.h;
    L.kind = !u.cont ? kPieceNormal : warm ? kPieceWarm : kPieceHead;
    L.spec_state = warm ? kNoState : spec;
    L.head_count = 0;
    L.done = 0;
    L.far = CP && u.cont && u.seg - (u.hs - P.origin) / (int64_t)P.seg_bytes > kContSpan;
    c.base = B.bytes + u.org;
    c.at = u.at;
    c.stop = warm ? u.lo_rel : min(u.hi_rel, u.limit);
    c.limit = u.limit;
    c.emit_from = warm ? 0xffffffffu : 0u;  // the warm-up reports nothing
    c.state = kRoot;
    c.have = 0;
    c.last_pid = c.last_end = 0;
    c.hay = u.h;
    c.hay_delta = (uint32_t)(u.org - u.hs);
    c.unit = (uint32_t)(2 * u.seg + 1);
    c.nemit = 0;
    c.cp_pos = u.at;
    c.cp_cont = 0;
}

// The current piece is finished (c.at >= c.stop, nothing pending): move on. Either starts the next
// piece (c.at = its first byte, c.state = its start state) or sets L.done and writes the segment summary.
template <int MODE, bool CP>
__device__ __forceinline__ void advance_piece(PieceCtx &c, LaneSeg &L, const Batch &B, const Sink &out, const SegOut &seg_out) {
    bool finish_segment = false;
    if (L.kind == kPieceWarm) {
        const uint32_t he_rel = c.limit;
        const uint32_t piece_end = min(L.hi_rel, he_rel);
        if (c.at == L.lo_rel) {
            // arrived at the segment start with a guess for the state there: scan the head piece from it
            L.spec_state = c.state;
            L.kind = kPieceHead;
            c.stop = piece_end;
            c.emit_from = 0;
            c.cp_pos = c.at;
            c.cp_cont = 0;
            return;
        }
        // a leftmost match kept the scanner busy past the segment start: no usable guess.
        // Leave the whole head piece to the repair pass.
        L.spec_state = kSpecSkipped;
        L.kind = kPieceHead;
        c.at = piece_end;
        c.stop = piece_end;
        c.emit_from = 0;
        c.state = kRoot;
        c.have = 0;
        c.cp_pos = L.lo_rel;  // its continuation bytes still have to be counted for the segments after it
        c.cp_cont = 0;
        // fall through: the (skipped) head piece is finished
    }
    if (L.kind == kPieceHead) L.head_count = c.nemit;
    if (c.stop == c.limit) {
        // the piece ended with its haystack: continue with the next non-empty haystack, if it starts inside the segment
        int64_t h = (int64_t)L.h + 1;
        while (h < B.n_haystacks && __ldg(B.offsets + h + 1) == __ldg(B.offsets + h)) h++;
        const int64_t hi_pos = L.org + L.hi_rel;
        if (h < B.n_haystacks && __ldg(B.offsets + h) < hi_pos) {
            const int64_t hs = __ldg(B.offsets + h), he = __ldg(B.offsets + h + 1);
            L.h = (uint32_t)h;
            L.kind = kPieceNormal;
            c.at = (uint32_t)(hs - L.org);
            c.limit = (uint32_t)(he - L.org);
            c.stop = min(L.hi_rel, c.limit);
            c.emit_from = 0;
            c.state = kRoot;
            c.have = 0;
            c.hay = (uint32_t)h;
            c.hay_delta = (uint32_t)(L.org - hs);
            c.cp_pos = c.at;
            c.cp_cont = 0;
            return;
        }
        finish_segment = true;
    } else {
        finish_segment = true;  // the segment ends inside this haystack
    }
    if (finish_segment) {
        uint32_t cont_tail = 0;
        if (CP) {
            // continuation bytes of the last piece inside the segment
            if (c.cp_pos <= L.hi_rel) {
                cp_catch_up(c, min(L.hi_rel, c.limit));
                cont_tail = c.cp_cont;
            } else {
                uint32_t n = c.cp_cont;
                for (uint32_t p = L.hi_rel; p < c.cp_pos; p++) n -= (ld_u8(c.base + p) & 0xC0u) == 0x80u;
                cont_tail = n;
            }
        }
        write_summary(seg_out, L.seg, L.spec_state, c.state, c.at - L.hi_rel, L.head_count, c.nemit, cont_tail, CP && L.far);
        L.done = 1;
    }
}

// Runs the exact scanner until the lane is at a point where the fast path can take over
// (hot state, nothing pending, inside a piece) or the segment is finished.
template <int MODE, bool CP>
__device__ __forceinline__ void settle(PieceCtx &c, LaneSeg &L, const DevImage &im, const Batch &B, const Sink &out,
                                    const SegOut &seg_out, HotMap hm, uint32_t min_at, bool stop_hot = true) {
    for (;;) {
        exact_scan<MODE, CP>(c, im, out, stop_hot, min_at, hm);
        if (c.at >= c.stop && (MODE != kModeLeftmost || !c.have)) {
            advance_piece<MODE, CP>(c, L, B, out, seg_out);
            if (L.done) return;
            min_at = c.at;
            continue;
        }
        return;
    }
}

template <int MODE, bool CP, int COLMODE, int V>
__global__ void __launch_bounds__((V == 1 ? kMaxWarps : kMaxWarps2) * 32, 1)
scan_staged_kernel(DevImage im, DevHot hot_img, Batch B, SegPlan P, Sink out, SegOut seg_out, uint32_t H,
                   uint32_t hot_bytes, unsigned int *task_counter, unsigned long long *trap_stats) {
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t hot_s = (uint32_t)__cvta_generic_to_shared(smem);  // the table; also the address of hot row 0 (the root)
    const uint32_t cmap_s = hot_s + hot_bytes;                        // 256 B
    const uint32_t bar_s = cmap_s + 256;                              // mbarrier, then the stream bounds (2 x int64)
    const uint32_t h2f_s = cmap_s + kStageOffset;                     // hot row -> automaton state, u32[H + 1] (the trap row maps to the dead state)
    const uint32_t stage_all_s = h2f_s + (((H + 1) * 4 + 127u) & ~127u);  // 128-aligned by construction
    const uint32_t row_entries = COLMODE == kColAscii ? kAsciiCols : im.n_cols;
    const uint32_t row_bytes = row_entries * 2;
    const uint32_t trap_off = H * row_bytes;
    const uint32_t trap = hot_s + trap_off;  // entries are shared ADDRESSES of rows (see the header comment)
    const uint16_t *src_table = COLMODE == kColAscii ? hot_img.table128 : hot_img.table;
    uint8_t *cmap = smem + hot_bytes;
    int64_t *bounds = reinterpret_cast<int64_t *>(smem + hot_bytes + 256 + 16);

    // ---- prologue: the hot table (L2 resident) ------------------------------------------
    const uint32_t n_entries = (H + 1) * row_entries;
    const uint32_t guard_entries = COLMODE == kColAscii ? kAsciiCols : 0;  // the speculative (unclamped) pass may read up to 254 bytes past the trap row
    uint32_t *tab32 = reinterpret_cast<uint32_t *>(smem);
    const uint32_t bias2 = hot_s | (hot_s << 16);
    if (H == (COLMODE == kColAscii ? hot_img.n_rows128 : hot_img.n_rows)) {
        // the whole image fits: one TMA bulk copy, completion on an mbarrier
        const uint32_t bytes = (n_entries * 2 + 15u) & ~15u;
        if (threadIdx.x == 0) {
            mbar_init(bar_s, 1);
            mbar_expect_tx(bar_s, bytes);
            tma_bulk_g2s(hot_s, src_table, bytes, bar_s);
            bounds[0] = __ldg(B.offsets);
            bounds[1] = __ldg(B.offsets + B.n_haystacks);
        }
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) cmap[i] = __ldg(im.colmap + i);
        __syncthreads();  // the barrier is initialised before anyone polls it
        mbar_wait(bar_s, 0);
        // offsets -> addresses (two entries per word; no carry: every address is below 64 K)
        for (uint32_t i = threadIdx.x; i < (n_entries + 1) / 2; i += blockDim.x) tab32[i] += bias2;
    } else {
        // a prefix of the image (rows are hottest-first): entries beyond it become the trap
        const uint32_t n = H * row_entries;
        const uint32_t *src32 = reinterpret_cast<const uint32_t *>(src_table);  // 16-byte aligned in the image
        for (uint32_t i = threadIdx.x; i < (n + 1) / 2; i += blockDim.x) {
            const uint32_t v = __ldg(src32 + i);
            tab32[i] = (min(v & 0xffffu, trap_off) | (min(v >> 16, trap_off) << 16)) + bias2;
        }
        __syncthreads();  // (an odd n: the word above also wrote the first trap-row entry; the fill below overwrites it)
        uint16_t *h16 = reinterpret_cast<uint16_t *>(smem);
        for (uint32_t i = threadIdx.x; i < row_entries; i += blockDim.x) h16[n + i] = (uint16_t)trap;
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) cmap[i] = __ldg(im.colmap + i);
        if (threadIdx.x == 0) {
            bounds[0] = __ldg(B.offsets);
            bounds[1] = __ldg(B.offsets + B.n_haystacks);
        }
    }
    {
        uint16_t *h16 = reinterpret_cast<uint16_t *>(smem);
        for (uint32_t i = threadIdx.x; i < guard_entries; i += blockDim.x) h16[n_entries + i] = (uint16_t)trap;
        uint32_t *h2f = reinterpret_cast<uint32_t *>(smem + hot_bytes + kStageOffset);
        for (uint32_t i = threadIdx.x; i <= H; i += blockDim.x) h2f[i] = i < H ? __ldg(hot_img.hot2full + i) : kDead;
    }
    __syncthreads();
    // 16-byte groups scanned, for the host's traps-per-group statistic (it re-profiles when traps are frequent)
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(trap_stats, (unsigned long long)((bounds[1] - bounds[0]) >> 4));

    HotMap hm;
    hm.full2hot = hot_img.full2hot;
    hm.hot_limit = H;
    FastTab ft;
    ft.cmap = cmap_s;
    ft.lo = im.col_lo;
    ft.maxc = im.n_cols - 1;
    // hot row index <-> row address
    auto row_of = [&](uint32_t addr) { return (addr - hot_s) / row_bytes; };
    // the automaton state of a hot row, from the shared-memory copy of hot2full (no global round trip on the
    // segment-end and warm-up-end paths)
    auto state_of = [&](uint32_t addr) { return lds32(h2f_s + row_of(addr) * 4); };

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr uint32_t kRows = 32 * V;                 // virtual lanes (segments) per warp-task
    constexpr uint32_t kBufBytes = kRows * kRow;       // one staging buffer of a warp
    constexpr uint32_t kWarpMeta = kRows * kMetaRow;
    const uint32_t meta_s = stage_all_s + warp * kWarpMeta;
    const uint32_t stage_s = stage_all_s + (blockDim.x >> 5) * kWarpMeta + warp * 2 * kBufBytes;
    const uintptr_t gbase = reinterpret_cast<uintptr_t>(B.bytes + P.origin);  // 64-byte aligned by construction of the plan
    // copy instruction i of a stage moves 16-byte unit (lane & 3) of row (i * 8 + lane / 4); the unit's
    // place in its row is swizzled by (row >> 1) & 3, which does not depend on i
    const uint32_t cp_dst = stage_s + (lane >> 2) * kRow + (((lane & 3) ^ ((lane >> 3) & 3)) << 4);
    const uint32_t cp_meta = meta_s + (lane >> 2) * kMetaRow;
    // this lane's rows (virtual lanes lane, lane + 32, ...): the address of unit 0 of the first
    const uint32_t row_s = stage_s + lane * kRow + (((lane >> 1) & 3) << 4);
    const uint32_t q = P.lane_stride;
    const uint32_t n_tasks = (uint32_t)(((uint64_t)P.n_segments + (uint64_t)kRows * q - 1) / ((uint64_t)kRows * q) * q);

    // The exact scanner's state and the segment bookkeeping live in LOCAL memory on purpose (their
    // addresses are laundered through an empty asm so the compiler cannot promote the ~28 words per
    // segment to registers): only the careful path touches them, and the chunk loop needs the registers.
    // They are built when a lane first hands over to the exact scanner (cold(), below), about 2 % of the
    // segments of config 2; until then a lane's state is its registers, its guessed start state in the
    // metadata row and the warp's task number in shared memory.
    PieceCtx c_mem[V];
    LaneSeg L_mem[V];
    PieceCtx *c_ptr = c_mem;
    LaneSeg *L_ptr = L_mem;
    asm volatile("" : "+l"(c_ptr), "+l"(L_ptr));
    const uint32_t task_s = bar_s + 128 + warp * 4;  // this warp's current task (not kept in a register across the chunk loop)

    // Warp-tasks (32 * V segments, lane_stride apart) come from an atomic counter.  The claim for the NEXT task
    // is issued when the last chunk of the current one starts: the atomic's round trip overlaps that chunk,
    // and the first bytes of the next task are pulled towards L2 meanwhile.  (Claiming a whole task ahead was
    // measured and is slower: a task claimed early by a busy warp cannot be taken by an idle one at the end.)
    unsigned int claimed = 0;
    if (lane == 0) claimed = atomicAdd(task_counter, 1u);
    for (;;) {
        const unsigned int task = __shfl_sync(0xffffffffu, claimed, 0);
        if (task >= n_tasks) break;

        // per segment of this lane (compile-time indexed: registers)
        uint32_t pos[V], s[V], stop[V], cpd[V];
        uint32_t hi_rel[V], stop_head[V];  // the segment end, and where the head piece (after the warm-up) stops
        bool done[V], warm[V];  // warm: the current piece is the silent warm-up before the segment
        bool cold[V];           // PieceCtx / LaneSeg have been built: from then on they are the segment's record
        uint32_t nch_max = 0;
        __syncwarp();  // the previous task no longer reads meta / the staging buffers
        if (lane == 0) sts32(task_s, task);
        const int64_t stream_lo = bounds[0], stream_hi = bounds[1];
#pragma unroll
        for (int t = 0; t < V; t++) {
            const SegSetup u = seg_setup<V>(P, B, stream_lo, stream_hi, gbase, task, (uint32_t)t * 32u + lane);
            if (u.outside) write_summary(seg_out, u.seg, kNoState, kRoot, 0u, 0u, 0u, 0u, false);  // nothing to scan
            // the first piece is never empty (lo < hi, and a warm-up starts before lo) and starts in the
            // root state, which is hot row 0: straight into the fast path
            pos[t] = u.at;
            s[t] = hot_s;
            stop[t] = u.cont ? u.lo_rel : min(u.hi_rel, u.limit);
            cpd[t] = 0;
            hi_rel[t] = u.hi_rel;
            stop_head[t] = min(u.hi_rel, u.limit);
            warm[t] = u.cont;
            done[t] = !u.live;
            cold[t] = false;
            const uint32_t nchunks = u.live ? (u.hi_rel + kChunk - 1) / kChunk : 0u;
            nch_max = max(nch_max, nchunks);
            // where each row's bytes are: read back by whichever lane copies them (no shuffles in the loop:
            // the compiler cannot prove the warp converged there and would emit a slow collective path)
            const uint32_t m = meta_s + ((uint32_t)t * 32u + lane) * kMetaRow;
            sts64(m, make_uint2(u.off16, nchunks));
            sts64(m + 8, make_uint2(kNoState, u.first_fetch));
        }
        const uint32_t kmax = __reduce_max_sync(0xffffffffu, nch_max);
        __syncwarp();
        // one segment per lane: the four rows this lane copies keep their (first unit, chunk count) in registers for
        // the whole task (two per lane: there are eight and the registers are needed elsewhere; they are re-read)
        uint2 mrow[4];
        if (V == 1) {
#pragma unroll
            for (int i = 0; i < 4; i++) mrow[i] = lds64(cp_meta + i * 8 * kMetaRow);
        }

        // stage chunk k of every row into buffer (k & 1)
        auto issue = [&](uint32_t k) {
            const uint32_t dst = cp_dst + (k & 1u) * kBufBytes;
#pragma unroll
            for (int i = 0; i < 4 * V; i++) {
                const uint2 m = V == 1 ? mrow[i & 3] : lds64(cp_meta + i * 8 * kMetaRow);
                const bool live = k < m.y;  // else the unit is zero-filled, from the grid origin (a valid address)
                const uint8_t *src = reinterpret_cast<const uint8_t *>(gbase) + (live ? (size_t)(m.x + k * 4 + (lane & 3)) << 4 : 0);
                if (reinterpret_cast<uintptr_t>(src) & 64)
                    cp_async16_last(dst + i * 8 * kRow, src, live ? 16u : 0u);
                else
                    cp_async16(dst + i * 8 * kRow, src, live ? 16u : 0u);
            }
            cp_async_commit();
        };
        // Chunk 0.  A row that starts with a warm-up fetches only the 16-byte units the scan reads (it starts at
        // the first warm-up byte; the units before it are zero-filled), sector by sector: the rest of that
        // 128-byte line is the end of the neighbouring segment, which another lane copies at another time, so
        // asking the L2 for the whole line (and dropping it first) would read it from DRAM twice.
        auto issue_first = [&]() {
#pragma unroll
            for (int i = 0; i < 4 * V; i++) {
                const uint2 m = lds64(cp_meta + i * 8 * kMetaRow);
                const uint32_t first = lds32v(cp_meta + i * 8 * kMetaRow + 12);
                const bool live = m.y != 0;
                const uint8_t *src = reinterpret_cast<const uint8_t *>(gbase) + (live ? (size_t)(m.x + (lane & 3)) << 4 : 0);
                if (first & kWarmFetch)
                    cp_async16_sector(cp_dst + i * 8 * kRow, src, live && (lane & 3) >= (first & 3u) ? 16u : 0u);
                else if (reinterpret_cast<uintptr_t>(src) & 64)
                    cp_async16_last(cp_dst + i * 8 * kRow, src, live ? 16u : 0u);
                else
                    cp_async16(cp_dst + i * 8 * kRow, src, live ? 16u : 0u);
            }
            cp_async_commit();
        };

        // Everything that is not a clean whole chunk, for segment t of this lane: 16-byte groups, then single
        // bytes; with tail set, what is left when the chunks are used up.  ONE instance of this code (t and
        // the row are run-time values here): it contains the exact scanner.
        auto careful = [&](uint32_t t, uint32_t relk, uint32_t row, bool tail) {
            PieceCtx &c = c_ptr[t];
            LaneSeg &L = L_ptr[t];
            // this segment's fast-path state, by value (the arrays stay compile-time indexed)
            uint32_t S = s[0], POS = pos[0], STOP = stop[0], CPD = cpd[0], HI = hi_rel[0], HEAD = stop_head[0];
            bool DONE = done[0], WARM = warm[0], COLD = cold[0];
#pragma unroll
            for (int u = 1; u < V; u++)
                if (t == (uint32_t)u) {
                    S = s[u];
                    POS = pos[u];
                    STOP = stop[u];
                    CPD = cpd[u];
                    HI = hi_rel[u];
                    HEAD = stop_head[u];
                    DONE = done[u];
                    WARM = warm[u];
                    COLD = cold[u];
                }
            const uint32_t spec_s = meta_s + (t * 32u + lane) * kMetaRow + 8;  // the guessed start state, until the record is built
            // hand the lane over to the exact scanner at position POS, come back at the next fast-resume point
            auto leave_fast = [&](uint32_t min_at) {
                if (!COLD) {
                    // the first time for this segment: build its record, as the fast path has left it
                    const SegSetup u = seg_setup<V>(P, B, bounds[0], bounds[1], gbase, lds32v(task_s), t * 32u + lane);
                    build_cold<CP>(c, L, u, P, B, WARM, lds32v(spec_s));
                    COLD = true;
                }
                c.state = state_of(S);
                c.at = POS;
                if (CP) {
                    c.cp_pos = POS;
                    c.cp_cont = CPD;
                }
                settle<MODE, CP>(c, L, im, B, out, seg_out, hm, min_at);
                DONE = L.done != 0;
                POS = c.at;
                STOP = c.stop;
                WARM = !DONE && L.kind == kPieceWarm;
                if (!DONE) {
                    S = hot_s + (uint32_t)__ldg(hot_img.full2hot + c.state) * row_bytes;
                    if (CP) {
                        cp_catch_up(c, POS);
                        CPD = c.cp_cont;
                    }
                }
            };
            // the piece ended exactly where the fast path stands: the cheap, common transitions
            // (warm-up -> head piece; end of the segment) without going through the exact scanner
            auto piece_end_fast = [&]() -> bool {
                if (WARM) {
                    // arrived at the segment start in state S: that is the guess; scan the head piece from it
                    STOP = HEAD;
                    if (COLD) {
                        L.spec_state = state_of(S);
                        L.kind = kPieceHead;
                        c.stop = STOP;
                        c.emit_from = 0;
                    } else {
                        sts32(spec_s, state_of(S));
                    }
                    CPD = 0;
                    WARM = false;
                    return true;
                }
                if (STOP == HI) {
                    // end of the segment: write the summary (everything it needs from local memory is read
                    // first, in one batch: the stores below would otherwise force re-reads)
                    if (COLD) {
                        const int64_t seg = L.seg;
                        const uint32_t nem = c.nemit, spec = L.spec_state, kind = L.kind, hc = L.head_count, far = L.far;
                        write_summary(seg_out, seg, spec, state_of(S), 0u, kind == kPieceHead ? nem : hc, nem, CP ? CPD : 0u, CP && far);
                        L.done = 1;
                    } else {
                        // nothing was reported: the guess, the end state and the continuation bytes are all there is
                        write_summary(seg_out, seg_of_lane<V>(P, lds32v(task_s), t * 32u + lane), lds32v(spec_s), state_of(S), 0u, 0u, 0u,
                                      CP ? CPD : 0u, false);
                    }
                    DONE = true;
                    return true;
                }
                return false;
            };
#pragma unroll 1
            for (int j = 0; j < (tail ? 1 : 4); j++) {
                const uint32_t g = relk + j * 16;
                if (!tail) {
                    if (DONE || POS < g || POS >= g + 16) continue;  // this lane is not inside this group
                    if (POS == g && g + 16 <= STOP) {
                        // a whole 16-byte group in the fast path
                        const uint4 w = lds128(row_unit(row, (uint32_t)j));
                        uint32_t x = fstep4<COLMODE>(S, w.x, ft);
                        x = fstep4<COLMODE>(x, w.y, ft);
                        x = fstep4<COLMODE>(x, w.z, ft);
                        x = fstep4<COLMODE>(x, w.w, ft);
                        if (x != trap) {
                            S = x;
                            POS += 16;
                            if (CP) {
                                if ((w.x | w.y | w.z | w.w) & 0x80808080u)
                                    CPD += cont_bytes(w.x) + cont_bytes(w.y) + cont_bytes(w.z) + cont_bytes(w.w);
                            }
                            continue;
                        }
                    }
                }
                // byte by byte through the hot table (bytes from the staged row): piece boundaries,
                // unaligned positions, and the group something happens in -- the exact scanner only
                // gets the byte that left the hot set (tail: no staged bytes are left to look at)
                while (!DONE && (tail || (POS >= g && POS < g + 16))) {
                    uint32_t min_at = STOP;
                    if (POS >= STOP) {
                        if (POS == STOP && piece_end_fast()) continue;
                    } else if (!tail) {
                        const uint32_t b = lds8(row_byte(row, POS - relk));
                        const uint32_t x = fstep<COLMODE>(S, b, ft);
                        if (x != trap) {
                            S = x;
                            POS++;
                            if (CP) CPD += (b & 0xC0u) == 0x80u;
                            continue;
                        }
                        atomicAdd(trap_stats + 1, 1ULL);  // how well the hot set fits the data: the host re-profiles when traps are frequent
                        min_at = POS + 1;
                    }
                    leave_fast(min_at);  // (the one place the exact scanner is entered from)
                }
            }
#pragma unroll
            for (int u = 0; u < V; u++)
                if (t == (uint32_t)u) {
                    s[u] = S;
                    pos[u] = POS;
                    stop[u] = STOP;
                    cpd[u] = CPD;
                    done[u] = DONE;
                    warm[u] = WARM;
                    cold[u] = COLD;
                }
        };

        // One chunk: each of the lane's segments that is in the clean middle of a piece takes its whole 64 bytes
        // through the table with one trap check -- the V dependent chains are independent of each other and
        // interleave, hiding each other's shared-memory latency; whatever is not clean goes the careful way.
        if (kmax)
            issue_first();
        else if (lane == 0)
            claimed = atomicAdd(task_counter, 1u);  // nothing to scan in this task (segments outside the stream)
        for (uint32_t k = 0; k <= kmax; k++) {
            const bool tail = k == kmax;  // past the last chunk: whatever is left of the segments (normally just their summaries)
            const uint32_t row0 = row_s + (k & 1u) * kBufBytes;
            const uint32_t relk = k * kChunk;
            if (!tail) {
                cp_async_wait_all();
                __syncwarp();
                if (k + 1 < kmax) {
                    issue(k + 1);
                } else if (lane == 0) {
                    claimed = atomicAdd(task_counter, 1u);  // the last chunk: fetch the next task meanwhile
                }
                bool clean[V], any_clean = false;
#pragma unroll
                for (int t = 0; t < V; t++) {
                    if (!done[t] && warm[t] && pos[t] == stop[t] && pos[t] == relk) {
                        // the warm-up ended right at this chunk, in state s: that is the guess for the segment start;
                        // the head piece is scanned from it (same as piece_end_fast in the careful path)
                        stop[t] = stop_head[t];
                        if (cold[t]) {
                            PieceCtx &c = c_ptr[t];
                            LaneSeg &L = L_ptr[t];
                            L.spec_state = state_of(s[t]);
                            L.kind = kPieceHead;
                            c.stop = stop[t];
                            c.emit_from = 0;
                        } else {
                            sts32(meta_s + ((uint32_t)t * 32u + lane) * kMetaRow + 8, state_of(s[t]));
                        }
                        cpd[t] = 0;
                        warm[t] = false;
                    }
                    clean[t] = !done[t] && pos[t] == relk && relk + kChunk <= stop[t];
                    any_clean |= clean[t];
                }
                if (any_clean) {
                    // (a segment that is not clean runs along on whatever its row holds; the result is discarded)
                    uint32_t x[V], hb[V];
                    uint4 w[V];
#pragma unroll
                    for (int t = 0; t < V; t++) {
                        x[t] = s[t];
                        hb[t] = 0;
                        w[t] = lds128(row0 + t * 32 * kRow);
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        uint4 wn[V];
#pragma unroll
                        for (int t = 0; t < V; t++) {
                            wn[t] = w[t];
                            if (j < 3) wn[t] = lds128(row_unit(row0 + t * 32 * kRow, (uint32_t)j + 1));  // in flight while unit j is scanned
                        }
#pragma unroll
                        for (int t = 0; t < V; t++) {
                            if (CP || COLMODE == kColAscii) hb[t] |= w[t].x | w[t].y | w[t].z | w[t].w;
                            if (COLMODE == kColAscii) {
                                // byte-indexed table: bytes >= 0x80 (rare in mostly-ASCII text) are folded onto column 127
                                // here, word-wise and only in the units that have any, so the chain needs no per-byte clamp
                                if ((w[t].x | w[t].y | w[t].z | w[t].w) & 0x80808080u) {
                                    w[t].x = clamp7f(w[t].x);
                                    w[t].y = clamp7f(w[t].y);
                                    w[t].z = clamp7f(w[t].z);
                                    w[t].w = clamp7f(w[t].w);
                                }
                            }
                        }
#pragma unroll
                        for (int t = 0; t < V; t++) x[t] = fstep4<COLMODE, false>(x[t], w[t].x, ft);
#pragma unroll
                        for (int t = 0; t < V; t++) x[t] = fstep4<COLMODE, false>(x[t], w[t].y, ft);
#pragma unroll
                        for (int t = 0; t < V; t++) x[t] = fstep4<COLMODE, false>(x[t], w[t].z, ft);
#pragma unroll
                        for (int t = 0; t < V; t++) x[t] = fstep4<COLMODE, false>(x[t], w[t].w, ft);
#pragma unroll
                        for (int t = 0; t < V; t++) w[t] = wn[t];
                    }
#pragma unroll
                    for (int t = 0; t < V; t++) {
                        const bool high = (hb[t] & 0x80808080u) != 0;
                        if (clean[t] && x[t] != trap) {
                            s[t] = x[t];
                            pos[t] += kChunk;
                            if (CP && high) {
                                // multi-byte characters in this chunk (rare in mostly-ASCII text): count their
                                // continuation bytes from the staged row again (do not keep 16 words live for this)
#pragma unroll
                                for (int j = 0; j < 4; j++) {
                                    const uint4 v = lds128(row_unit(row0 + t * 32 * kRow, (uint32_t)j));
                                    cpd[t] += cont_bytes(v.x) + cont_bytes(v.y) + cont_bytes(v.z) + cont_bytes(v.w);
                                }
                            }
                        }
                        // else: something happened in these 64 bytes; s and pos are untouched and the careful path
                        // goes through them group by group
                    }
                }
            }
            // segments that still stand inside this chunk (tail: that are not finished); a structured branch, so the
            // warp reconverges before the next chunk
            uint32_t need = 0;
#pragma unroll
            for (int t = 0; t < V; t++) need |= (!done[t] && (tail || pos[t] < relk + kChunk)) ? (1u << t) : 0u;
            if (need) {
#pragma unroll 1
                for (uint32_t t = 0; t < (uint32_t)V; t++)
                    if (need & (1u << t)) careful(t, relk, row0 + t * 32 * kRow, tail);
            }
        }
    }
}

}  // namespace acb
