// Microbenchmark behind DESIGN.md section 6: cycles per step of the scan kernel's dependent chain
//   LDS.U16 -> (IMAD | IDP4A) -> LDS.U16
// for 1..32 warps per SM and 1 or 2 independent chains per thread.  One CTA per SM, table of 40 KB of u16
// "row addresses" in shared memory, bytes from registers.  Build: nvcc -arch=sm_90a -O3 lds_chain.cu
#include <cstdint>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t lds_tab(uint32_t addr) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];\n" : "=r"(v) : "r"(addr)); return v; }
__device__ __forceinline__ uint32_t mad2(uint32_t col, uint32_t s) { uint32_t r; asm("mad.lo.u32 %0, %1, 2, %2;\n" : "=r"(r) : "r"(col), "r"(s)); return r; }
template <uint32_t K> __device__ __forceinline__ uint32_t dp(uint32_t s, uint32_t w) { uint32_t a; asm("dp4a.u32.u32 %0, %1, %2, %3;\n" : "=r"(a) : "r"(w), "r"(2u << (8 * K)), "r"(s)); return a; }

template <int MODE, int V, int SAME>  // SAME 1: every lane of a warp walks the same path (broadcast loads, no bank conflicts); MODE 0: PRMT + VIADDMNMX + IMAD + LDS (27 columns); 1: IDP4A + LDS (128 columns)
__global__ void chain(uint32_t *out, unsigned long long *cycles, int iters, uint32_t seed) {
    extern __shared__ uint16_t tab[];
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(tab);
    const uint32_t row_bytes = MODE == 0 ? 54 : 256, rows = MODE == 0 ? 740 : 156;
    for (uint32_t i = threadIdx.x; i < rows * row_bytes / 2; i += blockDim.x) {
        uint32_t h = (i * 2654435761u + seed) >> 7;
        tab[i] = (uint16_t)(base + (h % rows) * row_bytes);
    }
    __syncthreads();
    uint32_t s[V], w[V];
    for (int v = 0; v < V; v++) { s[v] = base; w[v] = ((SAME ? (threadIdx.x >> 5) : threadIdx.x) * 0x01010101u + seed + v * 7u) & 0x7f7f7f7fu; }
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int rep = 0; rep < 4; rep++) {
#pragma unroll
            for (int v = 0; v < V; v++) {
                if (MODE == 0) {
#pragma unroll
                    for (int k = 0; k < 4; k++) { uint32_t b = __byte_perm(w[v], 0, 0x4440 + k); uint32_t col = min(b - 97u, 26u); s[v] = lds_tab(mad2(col, s[v])); }
                }
            }
            if (MODE == 1) {
#pragma unroll
                for (int v = 0; v < V; v++) s[v] = lds_tab(dp<0>(s[v], w[v]));
#pragma unroll
                for (int v = 0; v < V; v++) s[v] = lds_tab(dp<1>(s[v], w[v]));
#pragma unroll
                for (int v = 0; v < V; v++) s[v] = lds_tab(dp<2>(s[v], w[v]));
#pragma unroll
                for (int v = 0; v < V; v++) s[v] = lds_tab(dp<3>(s[v], w[v]));
            }
#pragma unroll
            for (int v = 0; v < V; v++) w[v] = (w[v] * 1664525u + 1013904223u) & 0x7f7f7f7fu;
        }
    }
    const long long t1 = clock64();
    uint32_t acc = 0;
    for (int v = 0; v < V; v++) acc += s[v];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = (unsigned long long)(t1 - t0);
}

template <int MODE, int V, int SAME> void run(int warps, int sms) {
    uint32_t *out; unsigned long long *cyc;
    cudaMalloc(&out, sms * 1024 * 4); cudaMalloc(&cyc, sms * 8);
    const int iters = 2000;
    cudaFuncSetAttribute(chain<MODE, V, SAME>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    chain<MODE, V, SAME><<<sms, warps * 32, 41000>>>(out, cyc, iters, 12345u);
    chain<MODE, V, SAME><<<sms, warps * 32, 41000>>>(out, cyc, iters, 12345u);
    cudaDeviceSynchronize();
    std::vector<unsigned long long> h(sms);
    cudaMemcpy(h.data(), cyc, sms * 8, cudaMemcpyDeviceToHost);
    double avg = 0; for (auto c : h) avg += (double)c; avg /= sms;
    const double steps = (double)iters * 16;  // per chain
    printf("%s mode %d chains/thread %d warps %2d : %.1f cycles per step per chain, %.2f warp-steps per cycle per SM\n", SAME ? "lockstep" : "random  ", MODE, V, warps,
           avg / steps, steps * V * warps / avg);
    cudaFree(out); cudaFree(cyc);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount;
    for (int w : {1, 8, 16, 24, 32}) run<0, 1, 0>(w, sms);
    for (int w : {1, 8, 16, 24, 32}) run<1, 1, 0>(w, sms);
    for (int w : {8, 16, 22, 32}) run<0, 2, 0>(w, sms);
    for (int w : {8, 16, 22, 32}) run<1, 2, 0>(w, sms);
    for (int w : {1, 8, 16, 24, 32}) run<0, 1, 1>(w, sms);
    for (int w : {1, 8, 16, 24, 32}) run<1, 1, 1>(w, sms);
    for (int w : {8, 16, 22, 32}) run<0, 2, 1>(w, sms);
    for (int w : {8, 16, 22, 32}) run<1, 2, 1>(w, sms);
    return 0;
}
