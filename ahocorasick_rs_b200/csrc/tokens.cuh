// tokens.cuh -- the token-id byte format (acb_tokens_encode / acb_tokens_encode_host) and its encode kernel.
//
// A token id t, 0 <= t < ACB_TOKEN_ID_LIMIT (2^21), becomes exactly ACB_TOKEN_BYTES = 3 bytes:
//
//     b0 = 0x80 | (t >> 14)     b1 = (t >> 7) & 0x7f     b2 = t & 0x7f
//
// Only a token's first byte has its high bit set, and every encoded pattern starts with such a byte and is 3k bytes
// long, so every byte-level occurrence of an encoded pattern starts and ends on a token boundary: byte occurrences
// are token occurrences at start / 3, end / 3, one to one (DESIGN.md §4.12).  Plain little-endian ids lack this: with
// int32, pattern [1] = 01 00 00 00 occurs at byte 1 of [256, 0] = 00 01 00 00 00 00 00 00.
//
// token_code is the format's only statement; the kernel and the host encoder below both use it.
#pragma once
#include <stdint.h>

#include "../../include/acb200.h"

namespace acb {

// the three bytes of id t, little-endian in the low 24 bits (b0 | b1 << 8 | b2 << 16); t must be below 2^21
__host__ __device__ __forceinline__ uint32_t token_code(uint32_t t) {
    return (0x80u | (t >> 14)) | (((t >> 7) & 0x7fu) << 8) | ((t & 0x7fu) << 16);
}

// the inverse of token_code: the id whose three bytes are b0 b1 b2, or false when they are not a token's encoding
// (b0 without its high bit, or b1 / b2 with theirs)
__host__ __device__ __forceinline__ bool token_decode(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t &t) {
    if (b0 < 0x80u || b0 > 0xffu || b1 > 0x7fu || b2 > 0x7fu) return false;
    t = ((b0 & 0x7fu) << 14) | (b1 << 7) | b2;
    return true;
}

// the id of element i as a signed 64-bit value (uint16 ids are non-negative, int32 / int64 ids keep their sign)
template <typename T>
__host__ __device__ __forceinline__ long long token_value(T v) {
    return (long long)v;
}

__host__ __device__ __forceinline__ bool token_ok(long long v) { return v >= 0 && v < (long long)ACB_TOKEN_ID_LIMIT; }

constexpr int kTokGroup = 8;         // ids per thread and step: one 16-byte load of uint16, two of int32, four of int64
constexpr int kTokThreads = 256;

// 8 ids -> 24 bytes = 6 32-bit words (4 ids -> 3 words, twice)
__device__ __forceinline__ void token_store8(uint32_t *w, const uint32_t c[kTokGroup]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t c0 = c[4 * h], c1 = c[4 * h + 1], c2 = c[4 * h + 2], c3 = c[4 * h + 3];
        w[3 * h] = c0 | (c1 << 24);
        w[3 * h + 1] = (c1 >> 8) | (c2 << 16);
        w[3 * h + 2] = (c2 >> 16) | (c3 << 8);
    }
}

// VEC: the ids are 16-byte aligned and the output 4-byte aligned -- groups of 8 ids go through 16-byte loads and
// 32-bit stores.  Otherwise (misaligned views) every id is loaded alone and written as 3 byte stores.  The last
// n % 8 ids of the vector path are written by the first threads the same way.  A bad id lowers *bad to its index
// with atomicMin (one per group that holds one); its bytes are the low 21 bits' encoding and mean nothing.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kTokThreads) tokens_encode_kernel(const T *__restrict__ ids, unsigned long long n,
                                                                    uint8_t *__restrict__ out, unsigned long long *__restrict__ bad) {
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long scalar_from = 0;
    if (VEC) {
        const unsigned long long groups = n / kTokGroup;
        constexpr int kVecs = kTokGroup * (int)sizeof(T) / 16;   // 16-byte loads per group
        const uint4 *src = reinterpret_cast<const uint4 *>(ids);
        uint32_t *dst = reinterpret_cast<uint32_t *>(out);
        for (unsigned long long g = tid; g < groups; g += stride) {
            uint4 v[kVecs];
#pragma unroll
            for (int k = 0; k < kVecs; ++k) v[k] = __ldcs(src + g * kVecs + k);   // read once: stream past L2
            const T *e = reinterpret_cast<const T *>(v);
            uint32_t c[kTokGroup];
            int first_bad = kTokGroup;
#pragma unroll
            for (int k = kTokGroup - 1; k >= 0; --k) {
                const long long t = token_value(e[k]);
                if (!token_ok(t)) first_bad = k;
                c[k] = token_code((uint32_t)t & (ACB_TOKEN_ID_LIMIT - 1));
            }
            if (first_bad < kTokGroup) atomicMin(bad, g * kTokGroup + first_bad);
            uint32_t w[3 * kTokGroup / 4];
            token_store8(w, c);
#pragma unroll
            for (int k = 0; k < 3 * kTokGroup / 4; ++k) dst[g * (3 * kTokGroup / 4) + k] = w[k];
        }
        scalar_from = groups * kTokGroup;
    }
    for (unsigned long long i = scalar_from + tid; i < n; i += stride) {
        const long long t = token_value(ids[i]);
        if (!token_ok(t)) atomicMin(bad, i);
        const uint32_t c = token_code((uint32_t)t & (ACB_TOKEN_ID_LIMIT - 1));
        out[3 * i] = (uint8_t)c;
        out[3 * i + 1] = (uint8_t)(c >> 8);
        out[3 * i + 2] = (uint8_t)(c >> 16);
    }
}

// the host encoder (acb_tokens_encode_host): lowers *bad to the first bad index, like the kernel
template <typename T>
inline void token_encode_host(const T *ids, uint64_t n, uint8_t *out, uint64_t *bad) {
    uint64_t first_bad = *bad;
    for (uint64_t i = 0; i < n; ++i) {
        const long long t = token_value(ids[i]);
        if (!token_ok(t) && i < first_bad) first_bad = i;
        const uint32_t c = token_code((uint32_t)t & (ACB_TOKEN_ID_LIMIT - 1));
        out[3 * i] = (uint8_t)c;
        out[3 * i + 1] = (uint8_t)(c >> 8);
        out[3 * i + 2] = (uint8_t)(c >> 16);
    }
    *bad = first_bad;
}

}  // namespace acb
