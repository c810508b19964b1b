// Device helpers of the rotary position embedding, shared by rope.cu and the RoPE-fused instances of qk_norm.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "rope.h"

namespace b200 {

// Table row of token row t (t = b * tokens + j), or -1 for a prefix token.
__device__ __forceinline__ int rope_row(const RopeArgs& r, int t) {
    const int b = t / r.tokens, j = t - b * r.tokens;
    if (j < r.prefix) return -1;
    const int k = r.tokens - r.prefix;
    return r.keep ? __ldg(r.keep + static_cast<int64_t>(b) * k + (j - r.prefix)) : j - r.prefix;
}

// Rotates the four interleaved pairs of f (8 fp32 values, pairs p .. p + 3 of a head) by table row n: R, or its
// transpose R^T with kTranspose.  p is a multiple of 4, so the cos / sin of the four pairs are one 16-byte load each;
// the y / x split at pair hd / 4 lives in the tables, so a vector that straddles it needs nothing special.
template <bool kTranspose>
__device__ __forceinline__ void rope_rotate(float (&f)[8], const RopeArgs& r, int n, int half, int p) {
    const float4 c4 = __ldg(reinterpret_cast<const float4*>(r.cos + static_cast<int64_t>(n) * half + p));
    const float4 s4 = __ldg(reinterpret_cast<const float4*>(r.sin + static_cast<int64_t>(n) * half + p));
    const float c[4] = {c4.x, c4.y, c4.z, c4.w}, s[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float x0 = f[2 * q], x1 = f[2 * q + 1];
        if (kTranspose) {
            f[2 * q] = x0 * c[q] + x1 * s[q];
            f[2 * q + 1] = x1 * c[q] - x0 * s[q];
        } else {
            f[2 * q] = x0 * c[q] - x1 * s[q];
            f[2 * q + 1] = x1 * c[q] + x0 * s[q];
        }
    }
}

}  // namespace b200
