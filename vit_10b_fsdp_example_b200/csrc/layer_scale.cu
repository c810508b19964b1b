// LayerScale (CaiT; timm LayerScale, VisionTransformer(init_values=...)): a block branch u = a W^T + b is scaled per
// output channel, gamma o u.  The scale is folded into the layer instead of the activations:
//     gamma o (a W^T + b) = a (gamma o W)^T + gamma o b,   (gamma o W)[c, :] = gamma_c W[c, :],
// so the GEMM runs unchanged on Wg = bf16(gamma o W) and bg = bf16(gamma o b).  With dy' the gradient of the scaled
// branch, M = dy'^T a (the GEMM wgrad of the un-scaled layer) and S = colsum(dy'):
//     dW = gamma o M,  db = gamma o S,  dgamma_c = sum_r dy'[r, c] u[r, c] = sum_k W[c, k] M[c, k] + b_c S_c,
// and the dgrad is da = dy' Wg.  Both kernels therefore read the weight (and M) once, whatever the batch.
//
// One CTA owns row c of W [D, K]: dgamma_c is reduced in a fixed order (registers, warp shuffles, one shared-memory
// slot per warp), so it needs no atomics and is the same in every run.  Rows are streamed in 16-byte vectors from
// their first 16-byte boundary, with scalar head and tail elements; if W, Wg (and M) do not share their alignment
// modulo 16 bytes, every element is scalar.  Products and sums are fp32; each bf16 output is rounded once.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "layer_scale.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kLsThreads = 256;
constexpr int kLsUnroll = 4;  // 16-byte vectors per thread and array in flight

template <bool kBwd>
__global__ void __launch_bounds__(kLsThreads) layer_scale_kernel(
    const __nv_bfloat16* __restrict__ W, const __nv_bfloat16* __restrict__ b, const __nv_bfloat16* __restrict__ gamma,
    __nv_bfloat16* __restrict__ M, const float* __restrict__ S, __nv_bfloat16* __restrict__ Wg,
    __nv_bfloat16* __restrict__ bg, float* __restrict__ db, float* __restrict__ dgamma, int64_t K, bool vec) {
    const int64_t c = blockIdx.x;
    const float g = __bfloat162float(gamma[c]);
    const __nv_bfloat16* w = W + c * K;
    __nv_bfloat16* wg = Wg + c * K;
    __nv_bfloat16* m = kBwd ? M + c * K : nullptr;
    // Elements before the row's first 16-byte boundary (bf16 pointers are 2-byte aligned); all of them without vectors.
    const int64_t head = vec ? min(K, static_cast<int64_t>(((16 - (reinterpret_cast<uintptr_t>(w) & 15)) & 15) / 2)) : K;
    const int64_t nvec = (K - head) / 8;
    const int64_t tail = head + nvec * 8;
    float acc = 0.f;  // backward: this thread's part of sum_k W[c, k] M[c, k]

    auto scalar = [&](int64_t k) {
        const float x = __bfloat162float(w[k]);
        wg[k] = __float2bfloat16_rn(g * x);
        if constexpr (kBwd) {
            const float mk = __bfloat162float(m[k]);
            acc += x * mk;
            m[k] = __float2bfloat16_rn(g * mk);
        }
    };
    for (int64_t k = threadIdx.x; k < head; k += kLsThreads) scalar(k);
    for (int64_t k = tail + threadIdx.x; k < K; k += kLsThreads) scalar(k);

    const uint4* wv = reinterpret_cast<const uint4*>(w + head);
    uint4* gv = reinterpret_cast<uint4*>(wg + head);
    uint4* mv = kBwd ? reinterpret_cast<uint4*>(m + head) : nullptr;
    for (int64_t i0 = threadIdx.x; i0 < nvec; i0 += kLsThreads * kLsUnroll) {
        uint4 xv[kLsUnroll], mm[kLsUnroll];
#pragma unroll
        for (int u = 0; u < kLsUnroll; ++u) {
            const int64_t i = i0 + u * kLsThreads;
            xv[u] = i < nvec ? __ldg(wv + i) : make_uint4(0, 0, 0, 0);
            if constexpr (kBwd) mm[u] = i < nvec ? mv[i] : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < kLsUnroll; ++u) {
            const int64_t i = i0 + u * kLsThreads;
            if (i >= nvec) break;
            const uint32_t* xs = &xv[u].x;
            uint4 o;
            uint32_t* os = &o.x;
#pragma unroll
            for (int q = 0; q < 4; ++q) os[q] = pack_bf16x2(g * bf16_lo(xs[q]), g * bf16_hi(xs[q]));
            gv[i] = o;
            if constexpr (kBwd) {
                const uint32_t* ms = &mm[u].x;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float m0 = bf16_lo(ms[q]), m1 = bf16_hi(ms[q]);
                    acc += bf16_lo(xs[q]) * m0 + bf16_hi(xs[q]) * m1;
                    os[q] = pack_bf16x2(g * m0, g * m1);
                }
                mv[i] = o;
            }
        }
    }

    if constexpr (kBwd) {
        __shared__ float part[kLsThreads / 32];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (threadIdx.x % 32 == 0) part[threadIdx.x / 32] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < kLsThreads / 32; ++i) s += part[i];
            const float sc = S[c];
            dgamma[c] = s + __bfloat162float(b[c]) * sc;
            db[c] = g * sc;
        }
    } else if (threadIdx.x == 0) {
        bg[c] = __float2bfloat16_rn(g * __bfloat162float(b[c]));
    }
}

void check_ls(const char* what, int64_t D, int64_t K) {
    if (D < 1 || K < 1 || D > 0x7FFFFFFF)
        throw std::runtime_error(std::string(what) + ": need 1 <= D <= 2^31 - 1 rows and K >= 1 columns, got D " +
                                 std::to_string(D) + ", K " + std::to_string(K));
}

bool same_phase(const void* a, const void* b) {
    return ((reinterpret_cast<uintptr_t>(a) ^ reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}

inline void check_launch_ls(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

}  // namespace

void layer_scale_fold(const __nv_bfloat16* W, const __nv_bfloat16* b, const __nv_bfloat16* gamma, __nv_bfloat16* Wg,
                      __nv_bfloat16* bg, int64_t D, int64_t K, cudaStream_t stream) {
    check_ls("layer_scale_fold", D, K);
    layer_scale_kernel<false><<<static_cast<unsigned>(D), kLsThreads, 0, stream>>>(
        W, b, gamma, nullptr, nullptr, Wg, bg, nullptr, nullptr, K, same_phase(W, Wg));
    check_launch_ls("layer_scale_fold");
}

void layer_scale_bwd(const __nv_bfloat16* W, const __nv_bfloat16* b, const __nv_bfloat16* gamma, __nv_bfloat16* dW,
                     const float* S, __nv_bfloat16* Wg, float* db, float* dgamma, int64_t D, int64_t K,
                     cudaStream_t stream) {
    check_ls("layer_scale_bwd", D, K);
    layer_scale_kernel<true><<<static_cast<unsigned>(D), kLsThreads, 0, stream>>>(
        W, b, gamma, dW, S, Wg, nullptr, db, dgamma, K, same_phase(W, Wg) && same_phase(W, dW));
    check_launch_ls("layer_scale_bwd");
}

}  // namespace b200
