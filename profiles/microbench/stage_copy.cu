// Microbenchmark: the staged kernel's copy path with a stand-in for the scan.  Each lane of a warp owns one
// 1 KiB row (a segment); the rows of a warp-task lie lane_stride = 4 segments (4 KiB) apart, as in the kernel
// at config 2's defaults.  A warp copies 64 bytes per row per chunk with 16-byte cp.async (4 instructions per
// warp and chunk, the kernel's XOR swizzle), into a ring of 2 or 3 buffers, and then spins for a fixed time per
// chunk in place of the table walk.  32 warps per SM (one CTA), 400 k rows = 409.6 MB, tasks from an atomic
// counter.  Prints the time against the spin alone, and the share of warp time spent in cp.async.wait_group.
// Variants: the spin per chunk (the kernel's measured per-chunk time and half of it), the stage count, and the
// L2 prefetch-size qualifier of the copy.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 stage_copy.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

template <int PF>  // 0: cp.async.cg; 1: .L2::128B; 2: .L2::256B
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
    if (PF == 0) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
    if (PF == 1) asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
    if (PF == 2) asm volatile("cp.async.cg.shared.global.L2::256B [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

constexpr uint32_t kQ = 4, kSeg = 1024, kChunks = kSeg / 64, kBuf = 32 * 64;

template <int STAGES, int PF>
__global__ void __launch_bounds__(1024, 1) stage(const uint8_t *data, uint32_t n_rows, uint32_t spin, unsigned int *counter,
                                                 unsigned long long *stats, uint32_t *sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t stage = (uint32_t)__cvta_generic_to_shared(smem) + warp * STAGES * kBuf;
    const uint32_t n_tasks = n_rows / 32;
    uint32_t acc = 0;
    unsigned long long waited = 0;
    const long long t_start = clock64();
    for (;;) {
        unsigned int task = 0;
        if (lane == 0) task = atomicAdd(counter, 1u);
        task = __shfl_sync(0xffffffffu, task, 0);
        if (task >= n_tasks) break;
        // row r of the task: segment (task / q * 32 + r) * q + task % q
        const uint64_t seg0 = (uint64_t)(task / kQ) * 32 * kQ + task % kQ;
        auto issue = [&](uint32_t k) {
            if (k < kChunks) {
                const uint32_t buf = stage + (k % STAGES) * kBuf;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const uint32_t r = i * 8 + (lane >> 2);
                    const uint8_t *src = data + (seg0 + (uint64_t)r * kQ) * kSeg + k * 64 + (lane & 3) * 16;
                    cp_async16<PF>(buf + r * 64 + (((lane & 3) ^ ((r >> 1) & 3)) << 4), src);
                }
            }
            cp_commit();  // (an empty group past the last chunk keeps the wait count uniform)
        };
        for (uint32_t k = 0; k + 1 < STAGES; k++) issue(k);
        for (uint32_t k = 0; k < kChunks; k++) {
            const long long w0 = clock64();
            cp_wait<STAGES - 2>();
            __syncwarp();
            waited += (unsigned long long)(clock64() - w0);
            issue(k + STAGES - 1);
            uint32_t v;
            asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(stage + (k % STAGES) * kBuf + lane * 64));
            acc += v;
            const long long t0 = clock64();  // stand-in for the scan of the chunk
            while (clock64() - t0 < spin) {}
        }
        cp_wait<0>();
    }
    if (lane == 0) {
        atomicAdd(stats, waited);
        atomicAdd(stats + 1, (unsigned long long)(clock64() - t_start));
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

template <int STAGES, int PF> void run(const uint8_t *d, uint32_t rows, uint32_t spin, double clock_ghz, int sms) {
    unsigned int *ctr; unsigned long long *st; uint32_t *sink;
    cudaMalloc(&ctr, 4); cudaMalloc(&st, 16); cudaMalloc(&sink, 4);
    const size_t smem = (size_t)32 * STAGES * kBuf;
    cudaFuncSetAttribute(stage<STAGES, PF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    float best = 1e9; unsigned long long h[2] = {0, 0};
    for (int it = 0; it < 5; it++) {
        cudaMemset(ctr, 0, 4); cudaMemset(st, 0, 16);
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0);
        stage<STAGES, PF><<<sms, 32 * 32, smem>>>(d, rows, spin, ctr, st, sink);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) { best = ms; cudaMemcpy(h, st, 16, cudaMemcpyDeviceToHost); }
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    // the spin alone: chunks per warp (tasks spread evenly) x spin
    const double spin_ms = (double)rows / 32 / (sms * 32.0) * kChunks * spin / clock_ghz / 1e6;
    printf("stages %d %-9s spin %5u cyc: %.4f ms (spin alone %.4f), %6.1f GB/s, wait %.1f %% of warp time  (%s)\n", STAGES,
           PF == 0 ? "cg" : PF == 1 ? "L2::128B" : "L2::256B", spin, best, spin_ms, (double)rows * kSeg / best / 1e6,
           100.0 * h[0] / (double)h[1], cudaGetErrorString(cudaGetLastError()));
    cudaFree(ctr); cudaFree(st); cudaFree(sink);
}

template <int PF> void sweep(const uint8_t *d, uint32_t rows, uint32_t spin, double ghz, int sms) {
    run<2, PF>(d, rows, spin, ghz, sms);
    run<3, PF>(d, rows, spin, ghz, sms);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double ghz = khz / 1e6;
    const uint32_t rows = 400000;  // 100 k x 4 KiB haystacks cut into 1 KiB segments
    uint8_t *d; cudaMalloc(&d, (size_t)rows * kSeg); cudaMemset(d, 1, (size_t)rows * kSeg);
    printf("%s, %d SMs, max SM clock %.3f GHz\n", p.name, p.multiProcessorCount, ghz);
    // the kernel's time per chunk: 0.282 ms / ~50 chunks per warp = 5.6 us; and half of it
    for (double us : {5.6, 2.8, 0.0}) {
        const uint32_t spin = (uint32_t)(us * 1e3 * ghz);
        sweep<0>(d, rows, spin, ghz, p.multiProcessorCount);
        sweep<1>(d, rows, spin, ghz, p.multiProcessorCount);
        sweep<2>(d, rows, spin, ghz, p.multiProcessorCount);
    }
    cudaFree(d);
    return 0;
}
