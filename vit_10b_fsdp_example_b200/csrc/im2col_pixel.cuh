// The per-pixel fetch of the patch im2col, shared by im2col_kernel (elementwise.cu, every patch) and
// im2col_gather_kernel (patch_drop.cu, the kept patches of patch dropout), so both mix and index identically.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>

#include "elementwise.h"

namespace b200 {

// Column k < 3 P^2 (k = c * P * P + py * P + px) of patch `patch` = b * G * G + gy * G + gx (image b, grid G = S / P)
// from images [B, 3, S, S], with the batch mixing MIX of Im2colMix (0 none, 1 Mixup with image B-1-b, 2 CutMix box from
// image B-1-b).  Idx is the type of the patch index: int keeps the index math in 32 bits (no division calls).
template <typename T, int MIX, typename Idx>
__device__ __forceinline__ float im2col_pixel(const T* __restrict__ img, int B, int S, int P, int G, Idx patch, int k,
                                              const Im2colMix& mix) {
    const int c = k / (P * P), rem = k % (P * P), py = rem / P, px = rem % P;
    const int gx = static_cast<int>(patch % G), gy = static_cast<int>((patch / G) % G);
    const int64_t b = patch / (G * G);
    if constexpr (MIX == 0) {
        return static_cast<float>(img[((b * 3 + c) * S + gy * P + py) * S + gx * P + px]);
    } else {
        const int y = gy * P + py, x = gx * P + px;
        const int64_t pix = (static_cast<int64_t>(c) * S + y) * S + x, img_elems = 3LL * S * S;
        const int64_t b2 = B - 1 - b;
        if constexpr (MIX == 1) {
            const float a = static_cast<float>(img[b * img_elems + pix]);
            const float o = static_cast<float>(img[b2 * img_elems + pix]);
            return __fadd_rn(__fmul_rn(a, mix.lam), __fmul_rn(o, mix.mlam));
        } else {
            const bool in_box = y >= mix.yl && y < mix.yh && x >= mix.xl && x < mix.xh;
            return static_cast<float>(img[(in_box ? b2 : b) * img_elems + pix]);
        }
    }
}

}  // namespace b200
