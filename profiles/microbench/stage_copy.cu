// Microbenchmark: the staged kernel's copy path with a stand-in for the scan.  Each lane of a warp owns one
// 1 KiB row (a segment); the rows of a warp-task lie lane_stride = 4 segments (4 KiB) apart, as in the kernel
// at config 2's defaults.  A warp copies 64 bytes per row per chunk with 16-byte cp.async (4 instructions per
// warp and chunk, the kernel's XOR swizzle), into a ring of 2 or 3 buffers, and then spins for a fixed time per
// chunk in place of the table walk.  One CTA per SM, 400 k rows = 409.6 MB, tasks from an atomic counter.  Prints
// the time against the spin alone, and the share of warp time spent in cp.async.wait_group.
//
// The model (struct Model) also does what the kernel does besides copying and scanning, each part on its own switch:
//  - warm: 3 of every 4 segments (those that do not start a 4 KiB haystack) begin with a warm-up chunk, the 64 bytes
//    before the segment: 17 chunks instead of 16.  1: all four units, with the policy of any other chunk (the line
//    before the segment is fetched whole and, with evict_first, dropped first); 2: only the last 16 bytes, with a
//    plain cp.async.cg (one 32-byte sector);
//  - rec: each lane writes a record of `rec` words to local memory at task start and reads it back at the segment
//    end (28: the kernel's exact-scanner state and segment bookkeeping when every lane stores them; 6: the words
//    the segment end reads; 0: none, they are built only by lanes that need the exact scanner);
//  - summ: a 32-byte segment summary, 1: at the segment's own index (a warp's stores lie lane_stride * 32 B
//    apart), 2: at task * 32 + lane (a warp's stores are contiguous);
//  - claim: the next task is claimed when the last chunk starts.
// Levers on top of the full model (warm 1, rec 28, summ 1, claim): a bulk L2 prefetch (cp.async.bulk.prefetch.L2) of each lane's own next PFC chunks, PFD
// chunks ahead; the next task's first bytes prefetched during the current task's last chunk (claimed one chunk
// earlier); an evict_first L2 policy on the copies of chunks that complete their 128-byte line; 16 / 24 / 32 warps.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 stage_copy.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

template <int PF, bool EVF = false>  // PF 0: cp.async.cg; 1: .L2::128B; 2: .L2::256B.  EVF: with an L2 cache policy
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint64_t pol = 0) {
    if (EVF) {
        asm volatile("cp.async.cg.shared.global.L2::cache_hint.L2::128B [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "l"(pol) : "memory");
        return;
    }
    if (PF == 0) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
    if (PF == 1) asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
    if (PF == 2) asm volatile("cp.async.cg.shared.global.L2::256B [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;\n" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

constexpr uint32_t kQ = 4, kSeg = 1024, kBuf = 32 * 64, kRec = 28;  // kRec: u32 words of the per-lane local record

struct Model {
    int warm, rec, summ;
    bool claim;
};
constexpr Model kNone = {0, 0, 0, false}, kFull = {1, (int)kRec, 1, true};

struct Lever {
    Model model;
    int pfc, pfd;   // bulk L2 prefetch of the lane's next pfc chunks, pfd chunks ahead (pfc 0: none)
    bool next;      // the next task's first pfc (at least 4) chunks, during the last chunk
    bool evf;       // evict_first on copies that complete a 128-byte line
    int warps;
};

template <int STAGES, int PF, bool EVF>
__global__ void __launch_bounds__(1024, 1) stage(const uint8_t *data, uint32_t n_rows, uint32_t spin, Model md, int pfc, int pfd, bool next_pf,
                                                 unsigned int *counter, unsigned long long *stats, uint32_t *sink, uint4 *summaries) {
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t stage = (uint32_t)__cvta_generic_to_shared(smem) + warp * STAGES * kBuf;
    const uint32_t n_tasks = n_rows / 32;
    uint32_t acc = 0;
    unsigned long long waited = 0;
    uint64_t pol = 0;
    if (EVF) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
    uint32_t rec[kRec];  // local memory: the address is laundered so the record is not promoted to registers
    uint32_t *rp = rec;
    asm volatile("" : "+l"(rp));
    const long long t_start = clock64();
    unsigned int claimed = 0;
    if (md.claim && lane == 0) claimed = atomicAdd(counter, 1u);
    for (;;) {
        if (!md.claim && lane == 0) claimed = atomicAdd(counter, 1u);
        const unsigned int task = __shfl_sync(0xffffffffu, claimed, 0);
        if (task >= n_tasks) break;
        // row r of the task: segment (task / q * 32 + r) * q + task % q; a segment inside its haystack starts
        // with a warm-up chunk (all rows of a task alike)
        const uint64_t seg0 = (uint64_t)(task / kQ) * 32 * kQ + task % kQ;
        const bool warm = md.warm && task % kQ != 0;
        const uint32_t kmax = kSeg / 64 + (warm ? 1 : 0);
        const int64_t first = warm ? -64 : 0;  // of the row's first chunk, relative to its segment
#pragma unroll
        for (int i = 0; i < (int)kRec; i++)
            if (i < md.rec) rp[i] = (uint32_t)(seg0 + lane) * (i + 1);
        const uint8_t *mine = data + (int64_t)((seg0 + (uint64_t)lane * kQ) * kSeg) + first;
        auto issue = [&](uint32_t k) {
            if (k < kmax) {
                const uint32_t buf = stage + (k % STAGES) * kBuf;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const uint32_t r = i * 8 + (lane >> 2);
                    const uint8_t *src = data + (int64_t)((seg0 + (uint64_t)r * kQ) * kSeg) + first + k * 64 + (lane & 3) * 16;
                    const uint32_t dst = buf + r * 64 + (((lane & 3) ^ ((r >> 1) & 3)) << 4);
                    if (warm && k == 0 && md.warm == 2) {
                        if ((lane & 3) == 3) cp_async16<0>(dst, src);  // the unit the scan reads; the others are never looked at
                    } else if (EVF && (reinterpret_cast<uintptr_t>(src) & 64))
                        cp_async16<PF, true>(dst, src, pol);  // the second half of its 128-byte line: the line is spent
                    else
                        cp_async16<PF>(dst, src);
                }
            }
            cp_commit();  // (an empty group past the last chunk keeps the wait count uniform)
        };
        const uint32_t k_claim = next_pf ? kmax - 2 : kmax - 1;
        for (uint32_t k = 0; k + 1 < STAGES; k++) issue(k);
        for (uint32_t k = 0; k < kmax; k++) {
            const long long w0 = clock64();
            cp_wait<STAGES - 2>();
            __syncwarp();
            waited += (unsigned long long)(clock64() - w0);
            issue(k + STAGES - 1);
            if (md.claim && k == k_claim && lane == 0) claimed = atomicAdd(counter, 1u);
            if (pfc && k % pfc == 0 && k + pfd < kmax) {
                const uint32_t n = min((uint32_t)pfc, kmax - (k + pfd));
                prefetch_l2(mine + (k + pfd) * 64, n * 64);
            }
            if (next_pf && k == kmax - 1) {
                const unsigned int nt = __shfl_sync(0xffffffffu, claimed, 0);
                if (nt < n_tasks) {
                    const uint64_t ns = ((uint64_t)(nt / kQ) * 32 * kQ + nt % kQ) + (uint64_t)lane * kQ;
                    const int64_t nf = nt % kQ != 0 ? -64 : 0;
                    prefetch_l2(data + (int64_t)(ns * kSeg) + nf, max(pfc, 4) * 64);
                }
            }
            uint32_t v;
            asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(stage + (k % STAGES) * kBuf + lane * 64));
            acc += v;
            const long long t0 = clock64();  // stand-in for the scan of the chunk
            while (clock64() - t0 < spin) {}
        }
        // the segment end: the record read back, the summary written
        uint32_t x = 0;
#pragma unroll
        for (int i = 0; i < (int)kRec; i++)
            if (i < md.rec) x += rp[i];
        if (md.summ) {
            const uint64_t slot = md.summ == 2 ? (uint64_t)task * 32 + lane : seg0 + (uint64_t)lane * kQ;
            summaries[2 * slot] = make_uint4(x, acc, 0, 0);
            summaries[2 * slot + 1] = make_uint4(0, 0, x, 1);
        } else {
            acc += x;
        }
        cp_wait<0>();
    }
    if (lane == 0) {
        atomicAdd(stats, waited);
        atomicAdd(stats + 1, (unsigned long long)(clock64() - t_start));
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

template <int STAGES, int PF, bool EVF>
void run(const char *name, const uint8_t *d, uint32_t rows, uint32_t spin, double clock_ghz, int sms, Lever lv, uint4 *summ) {
    unsigned int *ctr; unsigned long long *st; uint32_t *sink;
    cudaMalloc(&ctr, 4); cudaMalloc(&st, 16); cudaMalloc(&sink, 4);
    const size_t smem = (size_t)lv.warps * STAGES * kBuf;
    cudaFuncSetAttribute(stage<STAGES, PF, EVF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    float best = 1e9, sum = 0; unsigned long long h[2] = {0, 0};
    const int iters = 20;
    for (int it = 0; it < iters + 2; it++) {
        cudaMemset(ctr, 0, 4); cudaMemset(st, 0, 16);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        stage<STAGES, PF, EVF><<<sms, lv.warps * 32, smem>>>(d, rows, spin, lv.model, lv.pfc, lv.pfd, lv.next, ctr, st, sink, summ);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (it >= 2) sum += ms;
        if (ms < best) { best = ms; cudaMemcpy(h, st, 16, cudaMemcpyDeviceToHost); }
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    // the spin alone: chunks per warp (tasks spread evenly) x spin
    const double chunks = lv.model.warm ? 16.75 : 16.0;
    const double spin_ms = (double)rows / 32 / (sms * lv.warps) * chunks * spin / clock_ghz / 1e6;
    printf("%-34s spin %5u cyc: best %.4f ms, mean %.4f (spin alone %.4f), %6.1f GB/s, wait %.1f %% of warp time  (%s)\n", name, spin,
           best, sum / iters, spin_ms, (double)rows * kSeg / best / 1e6, 100.0 * h[0] / (double)h[1], cudaGetErrorString(cudaGetLastError()));
    cudaFree(ctr); cudaFree(st); cudaFree(sink);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double ghz = khz / 1e6;
    const uint32_t rows = 400000;  // 100 k x 4 KiB haystacks cut into 1 KiB segments
    const int sms = p.multiProcessorCount;
    uint8_t *base; cudaMalloc(&base, (size_t)rows * kSeg + 256); cudaMemset(base, 1, (size_t)rows * kSeg + 256);
    const uint8_t *d = base + 128;  // room for the first segment's warm-up chunk
    uint4 *summ; cudaMalloc(&summ, (size_t)rows * 32);
    printf("%s, %d SMs, max SM clock %.3f GHz\n", p.name, sms, ghz);
    // the kernel's scan share per chunk: about half of its 4.8 us chunk period (0.240 ms / 49.6 chunks per warp);
    // 2.8 us is the spin of the earlier rows
    for (double us : {2.4, 2.8}) {
        const uint32_t spin = (uint32_t)(us * 1e3 * ghz);
        run<2, 1, false>("copies only, L2::128B", d, rows, spin, ghz, sms, {kNone, 0, 0, false, false, 32}, summ);
        run<2, 1, false>("model, L2::128B", d, rows, spin, ghz, sms, {kFull, 0, 0, false, false, 32}, summ);
        char name[64];
        for (int pfc : {2, 4, 8})
            for (int pfd : {1, 2, 4, 8}) {
                if (pfd < pfc / 2) continue;
                snprintf(name, sizeof name, "(a) R=%d D=%d", pfc * 64, pfd);
                run<2, 1, false>(name, d, rows, spin, ghz, sms, {kFull, pfc, pfd, false, false, 32}, summ);
            }
        run<2, 1, false>("(b) next task, 256 B", d, rows, spin, ghz, sms, {kFull, 0, 0, true, false, 32}, summ);
        run<2, 1, false>("(a)+(b) R=256 D=4", d, rows, spin, ghz, sms, {kFull, 4, 4, true, false, 32}, summ);
        run<2, 1, true>("(c) evict_first", d, rows, spin, ghz, sms, {kFull, 0, 0, false, true, 32}, summ);
        run<2, 1, true>("(a)+(b)+(c) R=256 D=4", d, rows, spin, ghz, sms, {kFull, 4, 4, true, true, 32}, summ);
        for (int w : {16, 24}) {
            snprintf(name, sizeof name, "(d) %d warps", w);
            run<2, 1, false>(name, d, rows, spin, ghz, sms, {kFull, 0, 0, false, false, w}, summ);
            snprintf(name, sizeof name, "(d) %d warps + (a)+(b) R=512 D=8", w);
            run<2, 1, false>(name, d, rows, spin, ghz, sms, {kFull, 8, 8, true, false, w}, summ);
        }
        // the parts of the model one at a time, on top of (c), which is what the kernel does: the full model first and
        // last (the spread between the two is the noise of this table)
        const Model parts[] = {kFull,          {2, 28, 1, true}, {0, 28, 1, true}, {1, 6, 1, true}, {1, 0, 1, true}, {1, 28, 2, true},
                               {1, 28, 0, true}, {1, 28, 1, false}, {2, 0, 1, true}, {2, 0, 2, true}, {0, 0, 0, true}, kFull};
        for (const Model &m : parts) {
            snprintf(name, sizeof name, "(c) warm %d rec %2d summ %d claim %d", m.warm, m.rec, m.summ, (int)m.claim);
            run<2, 1, true>(name, d, rows, spin, ghz, sms, {m, 0, 0, false, true, 32}, summ);
        }
    }
    cudaFree(base); cudaFree(summ);
    return 0;
}
