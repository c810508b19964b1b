// Memory-bound sm_90a kernels of the ViT training step: LayerNorm fwd/bwd, row softmax fwd/bwd,
// fused cross-entropy (loss + dlogits), patch im2col, bias-gradient column sums, sum of squares
// (grad-norm partials) and the fused sharded AdamW update.
//
// All of them are 128-bit vectorised, keep a row (or a thread's slice of it) in registers so DRAM is
// touched once per tensor, and accumulate in fp32.
//
// Capability parity (reference = ronghanghu/vit_10b_fsdp_example):
//   LayerNorm       -> timm Block.norm1/norm2 and FSDPViTModel.norm   (run_vit_training.py:134-141,151)
//   softmax         -> timm Attention                                  (run_vit_training.py:134)
//   cross entropy   -> torch.nn.CrossEntropyLoss                       (run_vit_training.py:229,262)
//   AdamW           -> torch.optim.AdamW over sharded params           (run_vit_training.py:237,278)
//   sum of squares  -> FSDP.clip_grad_norm_                            (run_vit_training.py:270)
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <stdexcept>
#include <string>

#include "dropout.cuh"
#include "elementwise.h"
#include "epilogue_math.cuh"
#include "im2col_pixel.cuh"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kLnThreads = 256;

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    f[0] = bf16_lo(v.x), f[1] = bf16_hi(v.x);
    f[2] = bf16_lo(v.y), f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z), f[5] = bf16_hi(v.z);
    f[6] = bf16_lo(v.w), f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 v;
    v.x = pack_bf16x2(f[0], f[1]);
    v.y = pack_bf16x2(f[2], f[3]);
    v.z = pack_bf16x2(f[4], f[5]);
    v.w = pack_bf16x2(f[6], f[7]);
    return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Sum over the whole CTA of up to two values at once. `red` is 2 * 32 floats of shared memory.
template <int kThreads>
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red) {
    a = warp_sum(a);
    b = warp_sum(b);
    const int w = threadIdx.x / 32, l = threadIdx.x % 32;
    __syncthreads();  // protect `red` from the previous use
    if (l == 0) {
        red[w] = a;
        red[32 + w] = b;
    }
    __syncthreads();
    float ra = (l < kThreads / 32) ? red[l] : 0.f;
    float rb = (l < kThreads / 32) ? red[32 + l] : 0.f;
    a = warp_sum(ra);
    b = warp_sum(rb);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: y = (x - mean) * rstd * gamma + beta ; saves mean / rstd per row.
// ------------------------------------------------------------------------------------------------
template <int kChunks>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ gamma,
                                                            const __nv_bfloat16* __restrict__ beta,
                                                            __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out,
                                                            float* __restrict__ rstd_out, int rows, int D, float eps) {
    __shared__ float red[64];
    const int nvec = D / 8;
    const float inv_d = 1.0f / static_cast<float>(D);
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
        const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<int64_t>(row) * D);
        uint4 v[kChunks];
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            v[i] = idx < nvec ? xr[idx] : make_uint4(0, 0, 0, 0);
        }
        float s = 0.f, dummy = 0.f;
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            float f[8];
            unpack8(v[i], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) s += f[q];
        }
        block_sum2<kLnThreads>(s, dummy, red);
        const float mean = s * inv_d;
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            if (idx < nvec) {
                float f[8];
                unpack8(v[i], f);
#pragma unroll
                for (int q = 0; q < 8; ++q) ss += (f[q] - mean) * (f[q] - mean);
            }
        }
        block_sum2<kLnThreads>(ss, dummy, red);
        const float rstd = rsqrtf(ss * inv_d + eps);
        if (threadIdx.x == 0) {
            mean_out[row] = mean;
            rstd_out[row] = rstd;
        }
        uint4* yr = reinterpret_cast<uint4*>(y + static_cast<int64_t>(row) * D);
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            if (idx < nvec) {
                float f[8], g[8], b[8];
                unpack8(v[i], f);
                unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + idx), g);
                unpack8(__ldg(reinterpret_cast<const uint4*>(beta) + idx), b);
#pragma unroll
                for (int q = 0; q < 8; ++q) f[q] = (f[q] - mean) * rstd * g[q] + b[q];
                yr[idx] = pack8(f);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward.  dx = [dres +] rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat))
// dgamma += sum_rows dy * xhat ; dbeta += sum_rows dy ; optionally dxsum += sum_rows dx
// (the latter is the bias gradient of the Linear that produced x's residual branch).
// A thread always owns the same columns, so the per-CTA column accumulators live in shared memory
// (plain read-modify-write, no atomics) instead of ~100 registers: 3 CTAs/SM stay resident and keep
// enough loads in flight to stream at HBM speed.
// ------------------------------------------------------------------------------------------------
template <int kChunks>
__global__ void __launch_bounds__(kLnThreads, 3) ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                               const __nv_bfloat16* __restrict__ x,
                                                               const __nv_bfloat16* __restrict__ gamma,
                                                               const float* __restrict__ mean_in,
                                                               const float* __restrict__ rstd_in,
                                                               const __nv_bfloat16* __restrict__ dres,
                                                               __nv_bfloat16* __restrict__ dx,
                                                               float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                               float* __restrict__ dxsum, int rows, int D) {
    __shared__ float red[64];
    extern __shared__ __align__(16) float acc[];  // [dg | db | dxs] each D floats
    float* acc_dg = acc;
    float* acc_db = acc + D;
    float* acc_dx = acc + 2 * D;
    const int nvec = D / 8;
    const float inv_d = 1.0f / static_cast<float>(D);
    const int narr = dxsum != nullptr ? 3 : 2;
    for (int i = threadIdx.x; i < narr * D; i += kLnThreads) acc[i] = 0.f;
    __syncthreads();
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
        const int64_t base = static_cast<int64_t>(row) * D;
        const uint4* xr = reinterpret_cast<const uint4*>(x + base);
        const uint4* dyr = reinterpret_cast<const uint4*>(dy + base);
        uint4 xv[kChunks], dv[kChunks];
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            xv[i] = idx < nvec ? xr[idx] : make_uint4(0, 0, 0, 0);
            dv[i] = idx < nvec ? dyr[idx] : make_uint4(0, 0, 0, 0);
        }
        const float mean = mean_in[row], rstd = rstd_in[row];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            if (idx < nvec) {
                float xf[8], df[8], gf[8];
                unpack8(xv[i], xf);
                unpack8(dv[i], df);
                unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + idx), gf);
                float4* pg = reinterpret_cast<float4*>(acc_dg + idx * 8);
                float4* pb = reinterpret_cast<float4*>(acc_db + idx * 8);
                float4 g0 = pg[0], g1 = pg[1], b0 = pb[0], b1 = pb[1];
                float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
                float ba[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float xhat = (xf[q] - mean) * rstd;
                    const float g = df[q] * gf[q];
                    s1 += g;
                    s2 += g * xhat;
                    ga[q] += df[q] * xhat;
                    ba[q] += df[q];
                }
                pg[0] = make_float4(ga[0], ga[1], ga[2], ga[3]);
                pg[1] = make_float4(ga[4], ga[5], ga[6], ga[7]);
                pb[0] = make_float4(ba[0], ba[1], ba[2], ba[3]);
                pb[1] = make_float4(ba[4], ba[5], ba[6], ba[7]);
            }
        }
        block_sum2<kLnThreads>(s1, s2, red);
        s1 *= inv_d;
        s2 *= inv_d;
        uint4* dxr = reinterpret_cast<uint4*>(dx + base);
#pragma unroll
        for (int i = 0; i < kChunks; ++i) {
            const int idx = threadIdx.x + i * kLnThreads;
            if (idx < nvec) {
                float xf[8], df[8], gf[8], rf[8], o[8];
                unpack8(xv[i], xf);
                unpack8(dv[i], df);
                unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + idx), gf);
                if (dres != nullptr) {
                    unpack8(reinterpret_cast<const uint4*>(dres + base)[idx], rf);
                } else {
#pragma unroll
                    for (int q = 0; q < 8; ++q) rf[q] = 0.f;
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float xhat = (xf[q] - mean) * rstd;
                    o[q] = rf[q] + rstd * (df[q] * gf[q] - s1 - xhat * s2);
                }
                const uint4 packed = pack8(o);
                dxr[idx] = packed;
                if (dxsum != nullptr) {
                    float ob[8];
                    unpack8(packed, ob);  // sum what was actually stored (bf16-rounded), like a torch .sum(0)
                    float4* px = reinterpret_cast<float4*>(acc_dx + idx * 8);
                    float4 a0 = px[0], a1 = px[1];
                    px[0] = make_float4(a0.x + ob[0], a0.y + ob[1], a0.z + ob[2], a0.w + ob[3]);
                    px[1] = make_float4(a1.x + ob[4], a1.y + ob[5], a1.z + ob[6], a1.w + ob[7]);
                }
            }
        }
    }
    // own columns only -> no intra-CTA hazard; one global atomic per column per CTA
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
        const int idx = threadIdx.x + i * kLnThreads;
        if (idx < nvec) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                atomicAdd(dgamma + idx * 8 + q, acc_dg[idx * 8 + q]);
                atomicAdd(dbeta + idx * 8 + q, acc_db[idx * 8 + q]);
                if (dxsum != nullptr) atomicAdd(dxsum + idx * 8 + q, acc_dx[idx * 8 + q]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm for narrow rows (D <= 2048): a row is handled by TPR threads (one 16 B vector each), a 256-thread CTA
// works on 256/TPR rows at once, and a thread keeps the column accumulators of its 8 columns in registers.
// The wide-row kernels above keep one row per CTA, which leaves most threads idle and serialises on two block
// barriers per row when D is only 1024 (ViT-L).
// ------------------------------------------------------------------------------------------------
template <int TPR>
__device__ __forceinline__ void group_sum2(float& a, float& b, float* red, int row_slot) {
    a = warp_sum(a);
    b = warp_sum(b);
    if constexpr (TPR > 32) {
        constexpr int kWarps = TPR / 32;
        const int w = (threadIdx.x % TPR) / 32, l = threadIdx.x % 32;
        __syncthreads();
        if (l == 0) {
            red[(row_slot * kWarps + w) * 2] = a;
            red[(row_slot * kWarps + w) * 2 + 1] = b;
        }
        __syncthreads();
        a = 0.f, b = 0.f;
#pragma unroll
        for (int i = 0; i < kWarps; ++i) {
            a += red[(row_slot * kWarps + i) * 2];
            b += red[(row_slot * kWarps + i) * 2 + 1];
        }
    }
}

template <int TPR>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_small_kernel(const __nv_bfloat16* __restrict__ x,
                                                                  const __nv_bfloat16* __restrict__ gamma,
                                                                  const __nv_bfloat16* __restrict__ beta,
                                                                  __nv_bfloat16* __restrict__ y,
                                                                  float* __restrict__ mean_out,
                                                                  float* __restrict__ rstd_out, int rows, int D,
                                                                  float eps) {
    __shared__ float red[2 * (kLnThreads / 32)];
    constexpr int kRowsPerCta = kLnThreads / TPR;
    const int nvec = D / 8;
    const int slot = threadIdx.x / TPR, idx = threadIdx.x % TPR;
    const bool active = idx < nvec;
    const float inv_d = 1.0f / static_cast<float>(D);
    float g[8], bta[8];
    if (active) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + idx), g);
        unpack8(__ldg(reinterpret_cast<const uint4*>(beta) + idx), bta);
    }
    const int iters = (rows + gridDim.x * kRowsPerCta - 1) / (gridDim.x * kRowsPerCta);
    for (int itn = 0; itn < iters; ++itn) {
        const int row = (itn * gridDim.x + blockIdx.x) * kRowsPerCta + slot;
        const bool ok = active && row < rows;
        float f[8];
        if (ok) {
            unpack8(reinterpret_cast<const uint4*>(x + static_cast<int64_t>(row) * D)[idx], f);
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] = 0.f;
        }
        float s = 0.f, dummy = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) s += f[q];
        group_sum2<TPR>(s, dummy, red, slot);
        const float mean = s * inv_d;
        float ss = 0.f;
        if (ok) {
#pragma unroll
            for (int q = 0; q < 8; ++q) ss += (f[q] - mean) * (f[q] - mean);
        }
        group_sum2<TPR>(ss, dummy, red, slot);
        const float rstd = rsqrtf(ss * inv_d + eps);
        if (ok) {
            if (idx == 0) {
                mean_out[row] = mean;
                rstd_out[row] = rstd;
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] = (f[q] - mean) * rstd * g[q] + bta[q];
            reinterpret_cast<uint4*>(y + static_cast<int64_t>(row) * D)[idx] = pack8(f);
        }
    }
}

template <int TPR>
__global__ void __launch_bounds__(kLnThreads) ln_bwd_small_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                  const __nv_bfloat16* __restrict__ x,
                                                                  const __nv_bfloat16* __restrict__ gamma,
                                                                  const float* __restrict__ mean_in,
                                                                  const float* __restrict__ rstd_in,
                                                                  const __nv_bfloat16* __restrict__ dres,
                                                                  __nv_bfloat16* __restrict__ dx,
                                                                  float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                  float* __restrict__ dxsum, int rows, int D) {
    __shared__ float red[2 * (kLnThreads / 32)];
    constexpr int kRowsPerCta = kLnThreads / TPR;
    const int nvec = D / 8;
    const int slot = threadIdx.x / TPR, idx = threadIdx.x % TPR;
    const bool active = idx < nvec;
    const float inv_d = 1.0f / static_cast<float>(D);
    float gam[8], dg[8], db[8], dxs[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) gam[q] = 0.f, dg[q] = 0.f, db[q] = 0.f, dxs[q] = 0.f;
    if (active) unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + idx), gam);
    const int iters = (rows + gridDim.x * kRowsPerCta - 1) / (gridDim.x * kRowsPerCta);
    for (int itn = 0; itn < iters; ++itn) {
        const int row = (itn * gridDim.x + blockIdx.x) * kRowsPerCta + slot;
        const bool ok = active && row < rows;
        const int64_t base = static_cast<int64_t>(row) * D;
        float xf[8], df[8], rf[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) xf[q] = 0.f, df[q] = 0.f, rf[q] = 0.f;
        float mean = 0.f, rstd = 0.f;
        if (ok) {
            unpack8(reinterpret_cast<const uint4*>(x + base)[idx], xf);
            unpack8(reinterpret_cast<const uint4*>(dy + base)[idx], df);
            if (dres != nullptr) unpack8(reinterpret_cast<const uint4*>(dres + base)[idx], rf);
            mean = mean_in[row];
            rstd = rstd_in[row];
        }
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float xhat = (xf[q] - mean) * rstd;
            const float gq = df[q] * gam[q];
            s1 += gq;
            s2 += gq * xhat;
            dg[q] += df[q] * xhat;
            db[q] += df[q];
        }
        group_sum2<TPR>(s1, s2, red, slot);
        s1 *= inv_d;
        s2 *= inv_d;
        if (ok) {
            float o[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float xhat = (xf[q] - mean) * rstd;
                o[q] = rf[q] + rstd * (df[q] * gam[q] - s1 - xhat * s2);
            }
            const uint4 packed = pack8(o);
            reinterpret_cast<uint4*>(dx + base)[idx] = packed;
            if (dxsum != nullptr) {
                float ob[8];
                unpack8(packed, ob);
#pragma unroll
                for (int q = 0; q < 8; ++q) dxs[q] += ob[q];
            }
        }
    }
    // combine the row slots of this CTA in shared memory, then one global atomic per column per CTA
    // (per-address atomics serialise in L2: 1776 -> ~300 arrivals per address for ViT-L)
    extern __shared__ __align__(16) float comb[];  // [3][TPR * 8]
    constexpr int kCols = TPR * 8;
    for (int i = threadIdx.x; i < 3 * kCols; i += kLnThreads) comb[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        atomicAdd(&comb[idx * 8 + q], dg[q]);
        atomicAdd(&comb[kCols + idx * 8 + q], db[q]);
        if (dxsum != nullptr) atomicAdd(&comb[2 * kCols + idx * 8 + q], dxs[q]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < D; c += kLnThreads) {
        atomicAdd(dgamma + c, comb[c]);
        atomicAdd(dbeta + c, comb[kCols + c]);
        if (dxsum != nullptr) atomicAdd(dxsum + c, comb[2 * kCols + c]);
    }
}

// ------------------------------------------------------------------------------------------------
// Stand-alone exact GELU / dGELU.  For short-K GEMMs (ViT-L: K = 1024) the activation math does not fit under the
// MMA time of a tile, so the fused epilogue would run the tensor cores at half speed; the op layer then uses the
// plain GEMM plus these memory-bound kernels (for ViT-10B, K = 5120, the activations stay fused in the epilogue).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gelu_fwd_kernel(const __nv_bfloat16* __restrict__ u, __nv_bfloat16* __restrict__ g,
                                                       int64_t nvec) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float f[8];
        unpack8(reinterpret_cast<const uint4*>(u)[i], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float e;
            f[q] = 0.5f * f[q] * (1.0f + erf_poly(f[q] * 0.70710678118654752f, e));
        }
        reinterpret_cast<uint4*>(g)[i] = pack8(f);
    }
}

__global__ void __launch_bounds__(256) dgelu_mul_kernel(const __nv_bfloat16* __restrict__ dg,
                                                        const __nv_bfloat16* __restrict__ u,
                                                        __nv_bfloat16* __restrict__ du, int64_t nvec) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        float f[8], d[8];
        unpack8(reinterpret_cast<const uint4*>(u)[i], f);
        unpack8(reinterpret_cast<const uint4*>(dg)[i], d);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float e;
            const float cdf = 0.5f * (1.0f + erf_poly(f[q] * 0.70710678118654752f, e));
            d[q] *= fmaf(f[q] * 0.3989422804014327f, e, cdf);
        }
        reinterpret_cast<uint4*>(du)[i] = pack8(d);
    }
}

// ------------------------------------------------------------------------------------------------
// Stand-alone SwiGLU (timm SwiGLUPacked): u = [gate | value] [M, 2H'], g = silu(gate) * value [M, H'].  The short-K
// counterparts of the GEMM's SwiGLU / dSwiGLU epilogues, and the re-materialisation of g in backward.  One thread owns 8
// adjacent columns of one row (16-byte vectors of the gate, the value and the output); sigmoid is the GEMM epilogue's
// sigmoid_approx (epilogue_math.cuh), so the fused and unfused routes compute the same function.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ u,
                                                         __nv_bfloat16* __restrict__ g, int64_t M, int hvec) {
    // rows over grid.y, 16-byte column vectors over grid.x: no 64-bit division (it would be a subroutine call)
    for (int64_t row = blockIdx.y; row < M; row += gridDim.y)
        for (int cv = blockIdx.x * blockDim.x + threadIdx.x; cv < hvec; cv += gridDim.x * blockDim.x) {
        const int64_t i = row * hvec + cv;
        const uint4* ur = reinterpret_cast<const uint4*>(u) + row * 2 * hvec;
        float a[8], b[8];
        unpack8(ur[cv], a);
        unpack8(ur[hvec + cv], b);
#pragma unroll
        for (int q = 0; q < 8; ++q) b[q] *= a[q] * sigmoid_approx(a[q]);
        reinterpret_cast<uint4*>(g)[i] = pack8(b);
    }
}

__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ dg,
                                                         const __nv_bfloat16* __restrict__ u,
                                                         __nv_bfloat16* __restrict__ du, int64_t M, int hvec) {
    // rows over grid.y, 16-byte column vectors over grid.x: no 64-bit division (it would be a subroutine call)
    for (int64_t row = blockIdx.y; row < M; row += gridDim.y)
        for (int cv = blockIdx.x * blockDim.x + threadIdx.x; cv < hvec; cv += gridDim.x * blockDim.x) {
        const int64_t i = row * hvec + cv;
        const uint4* ur = reinterpret_cast<const uint4*>(u) + row * 2 * hvec;
        float a[8], b[8], d[8];
        unpack8(ur[cv], a);
        unpack8(ur[hvec + cv], b);
        unpack8(reinterpret_cast<const uint4*>(dg)[i], d);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float s = sigmoid_approx(a[q]);
            const float dq = d[q];
            d[q] = dq * b[q] * (s * fmaf(a[q], 1.0f - s, 1.0f));  // du_gate = dg * b * silu'(a)
            b[q] = dq * (a[q] * s);                               // du_val  = dg * silu(a)
        }
        uint4* dr = reinterpret_cast<uint4*>(du) + row * 2 * hvec;
        dr[cv] = pack8(d);
        dr[hvec + cv] = pack8(b);
    }
}

// ------------------------------------------------------------------------------------------------
// Dropout on the kernel path (reference flags --pos_dropout / --att_dropout / --mlp_dropout, run_vit_training.py:
// 345-347): y = x * keep / (1 - p) with keep drawn from Philox-4x32-10, counter = index of the 16-byte vector, key =
// the 64-bit (seed, step, site) key of the engine's DropoutCtx.  The mask is a pure function of (key, element index),
// so the activation-checkpoint recompute and the backward pass regenerate it instead of storing it: one Philox call
// yields 8 x 16 random bits = the 8 bf16 values of a vector (keep <=> r16 >= p * 65536).  philox4x32_10 and the
// threshold live in dropout.cuh: the fused attention kernels regenerate the same mask for attention dropout.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dropout_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                      int64_t nvec, uint32_t key_lo, uint32_t key_hi, uint32_t thresh16,
                                                      float scale) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        uint32_t r[4];
        philox4x32_10(static_cast<uint32_t>(i), static_cast<uint32_t>(i >> 32), key_lo, key_hi, r);
        float f[8];
        unpack8(reinterpret_cast<const uint4*>(x)[i], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint32_t r16 = (r[q >> 1] >> ((q & 1) * 16)) & 0xFFFFu;
            f[q] = r16 >= thresh16 ? f[q] * scale : 0.f;
        }
        reinterpret_cast<uint4*>(y)[i] = pack8(f);
    }
}

// ------------------------------------------------------------------------------------------------
// Stochastic depth (timm drop_path): one keep / drop draw per sample of a residual branch.  Sample g (the global index
// sample_offset + b, so that ranks draw disjoint samples) is kept iff keep bit g % 8 of dropout_keep8(g / 8, key,
// thresh16) is set: the same Philox stream, 16-bit quantisation and scale as the dropout kernel, so the effective keep
// probability is 1 - thresh16 / 65536.  The per-sample scale vector (0 or dropout_scale) feeds the row scale of the
// branch's last GEMM in the forward and drop_path_bwd in the backward.
// ------------------------------------------------------------------------------------------------
__global__ void drop_path_scale_kernel(float* __restrict__ scale, int B, int64_t sample_offset, uint32_t key_lo,
                                       uint32_t key_hi, uint32_t thresh16, float keep_scale) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint64_t g = static_cast<uint64_t>(sample_offset) + static_cast<uint64_t>(b);
    const uint32_t bits = dropout_keep8(g / 8, key_lo, key_hi, thresh16);
    scale[b] = ((bits >> (g % 8)) & 1u) ? keep_scale : 0.f;
}

// dt = bf16(scale[row / N] * dy) and fp32 column sums of the rounded dt (the bias gradient of the branch's last linear
// layer) in one pass.  Same layout as colsum_kernel: a thread owns one 8-column vector of a slab of rows; four rows are
// loaded before any is processed so that each thread keeps four 16-byte loads in flight.
__global__ void __launch_bounds__(256) drop_path_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                            const float* __restrict__ scale,
                                                            __nv_bfloat16* __restrict__ dt, float* __restrict__ colsum,
                                                            int64_t rows, int C, int N, int rows_per_cta) {
    const int vec = blockIdx.x * blockDim.x + threadIdx.x;
    if (vec * 8 >= C) return;
    const int64_t r0 = static_cast<int64_t>(blockIdx.y) * rows_per_cta;
    const int64_t r1 = min(rows, r0 + rows_per_cta);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    auto row = [&](const uint4& in, int64_t r) {
        const float s = __ldg(scale + r / N);
        float f[8];
        unpack8(in, f);
#pragma unroll
        for (int q = 0; q < 8; ++q) f[q] *= s;
        const uint4 out = pack8(f);
        *reinterpret_cast<uint4*>(dt + r * C + vec * 8) = out;
        unpack8(out, f);  // the column sums are those of the rounded gradient the GEMMs consume
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
    };
    int64_t r = r0;
    for (; r + 4 <= r1; r += 4) {
        uint4 in[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) in[u] = __ldg(reinterpret_cast<const uint4*>(dy + (r + u) * C + vec * 8));
#pragma unroll
        for (int u = 0; u < 4; ++u) row(in[u], r + u);
    }
    for (; r < r1; ++r) row(__ldg(reinterpret_cast<const uint4*>(dy + r * C + vec * 8)), r);
#pragma unroll
    for (int q = 0; q < 8; ++q) atomicAdd(colsum + vec * 8 + q, acc[q]);
}

// ------------------------------------------------------------------------------------------------
// Token mean-pool of the head (reference run_vit_training.py:161: x.mean(dim=1) after the final norm) and its backward.
// Forward: pooled[b, :] = mean_n xn[b, n, :] -- a CTA column-strip sums the N tokens of one image in fp32.
// Backward: d xn[b, n, :] = dpooled[b, :] / N for every token; written as the broadcast rows the final-LayerNorm
// backward consumes (one pass, no [B, N, D] fp32 intermediate as in the eager expand + div).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) meanpool_fwd_kernel(const __nv_bfloat16* __restrict__ xn,
                                                           __nv_bfloat16* __restrict__ pooled, int N, int D) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;  // 16-byte vector (8 columns)
    if (v >= D / 8) return;
    const uint4* src = reinterpret_cast<const uint4*>(xn + static_cast<int64_t>(b) * N * D) + v;
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    int n = 0;
    for (; n + 4 <= N; n += 4) {  // 4 independent loads in flight
        uint4 t[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) t[u] = src[static_cast<int64_t>(n + u) * (D / 8)];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            float f[8];
            unpack8(t[u], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += f[q];
        }
    }
    for (; n < N; ++n) {
        float f[8];
        unpack8(src[static_cast<int64_t>(n) * (D / 8)], f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
    }
    const float inv = 1.0f / static_cast<float>(N);
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] *= inv;
    reinterpret_cast<uint4*>(pooled + static_cast<int64_t>(b) * D)[v] = pack8(acc);
}

__global__ void __launch_bounds__(128) meanpool_bwd_kernel(const __nv_bfloat16* __restrict__ dpooled,
                                                           __nv_bfloat16* __restrict__ dxn, int N, int D) {
    const int b = blockIdx.y;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= D / 8) return;
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(dpooled + static_cast<int64_t>(b) * D)[v], f);
    const float inv = 1.0f / static_cast<float>(N);
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] *= inv;
    const uint4 o = pack8(f);
    uint4* dst = reinterpret_cast<uint4*>(dxn + static_cast<int64_t>(b) * N * D) + v;
    for (int n = 0; n < N; ++n) dst[static_cast<int64_t>(n) * (D / 8)] = o;
}

// ------------------------------------------------------------------------------------------------
// Row softmax (attention probabilities), in place on a [rows, ld] bf16 matrix with `n` valid columns.
// One warp per row; fp32 math; exp2 with pre-multiplied log2(e).
// ------------------------------------------------------------------------------------------------
template <int kMaxPairs>  // bf16x2 pairs per lane
__global__ void softmax_fwd_kernel(__nv_bfloat16* __restrict__ s, int64_t rows, int n, int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    uint32_t* r = reinterpret_cast<uint32_t*>(s + row * ld);
    const int npairs = n / 2;
    const float sl2 = scale * 1.4426950408889634f;
    float v[kMaxPairs][2];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < kMaxPairs; ++i) {
        const int idx = lane + i * 32;
        if (idx < npairs) {
            const uint32_t w = r[idx];
            v[i][0] = bf16_lo(w) * sl2;
            v[i][1] = bf16_hi(w) * sl2;
            mx = fmaxf(mx, fmaxf(v[i][0], v[i][1]));
        } else {
            v[i][0] = v[i][1] = -INFINITY;
        }
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPairs; ++i) {
        v[i][0] = exp2f(v[i][0] - mx);
        v[i][1] = exp2f(v[i][1] - mx);
        sum += v[i][0] + v[i][1];
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < kMaxPairs; ++i) {
        const int idx = lane + i * 32;
        if (idx < npairs) r[idx] = pack_bf16x2(v[i][0] * inv, v[i][1] * inv);
    }
}

// dS = scale * P * (dP - sum_j dP_j P_j), in place on dP.
template <int kMaxPairs>
__global__ void softmax_bwd_kernel(__nv_bfloat16* __restrict__ dp, const __nv_bfloat16* __restrict__ p, int64_t rows,
                                   int n, int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    uint32_t* dr = reinterpret_cast<uint32_t*>(dp + row * ld);
    const uint32_t* pr = reinterpret_cast<const uint32_t*>(p + row * ld);
    const int npairs = n / 2;
    float pv[kMaxPairs][2], dv[kMaxPairs][2];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPairs; ++i) {
        const int idx = lane + i * 32;
        if (idx < npairs) {
            const uint32_t a = pr[idx], b = dr[idx];
            pv[i][0] = bf16_lo(a), pv[i][1] = bf16_hi(a);
            dv[i][0] = bf16_lo(b), dv[i][1] = bf16_hi(b);
            dot += pv[i][0] * dv[i][0] + pv[i][1] * dv[i][1];
        } else {
            pv[i][0] = pv[i][1] = dv[i][0] = dv[i][1] = 0.f;
        }
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int i = 0; i < kMaxPairs; ++i) {
        const int idx = lane + i * 32;
        if (idx < npairs)
            dr[idx] = pack_bf16x2(scale * pv[i][0] * (dv[i][0] - dot), scale * pv[i][1] * (dv[i][1] - dot));
    }
}

// ------------------------------------------------------------------------------------------------
// Row softmax fwd / bwd for the rows the pair kernels above do not take: odd n (an odd patch grid, e.g. 7 x 7 or
// 37 x 37 tokens) and n > 1024.  Same math (fp32, exp2 with the scale folded in), one warp per row, 16-byte vectors:
// ld must be a multiple of 8.  The last vector of a row may be partial; its columns n..ld-1 are padding, masked on
// load and never written.  Up to n = 2048 the row stays in registers (kVecs vectors per lane); longer rows stream
// twice through L1/L2: online max / sum (fwd) or the dot product (bwd), then the write.
// ------------------------------------------------------------------------------------------------
constexpr int kSoftmaxRegMaxN = 32 * 8 * 8;

// Scores of vector `idx` of a row, times sl2; columns >= n become -inf.
__device__ __forceinline__ void load_scores8(const __nv_bfloat16* r, int idx, int n, float sl2, float (&f)[8]) {
    unpack8(reinterpret_cast<const uint4*>(r)[idx], f);
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] = idx * 8 + q < n ? f[q] * sl2 : -INFINITY;
}

// Vector `idx` of a row; columns >= n read as 0.
__device__ __forceinline__ void load_masked8(const __nv_bfloat16* r, int idx, int n, float (&f)[8]) {
    unpack8(reinterpret_cast<const uint4*>(r)[idx], f);
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] = idx * 8 + q < n ? f[q] : 0.f;
}

// Writes the columns < n of vector `idx`: one 16-byte store, or element stores for the partial last vector.
__device__ __forceinline__ void store_row8(__nv_bfloat16* r, int idx, int n, const float (&f)[8]) {
    if (idx * 8 + 8 <= n) {
        reinterpret_cast<uint4*>(r)[idx] = pack8(f);
    } else {
#pragma unroll
        for (int q = 0; q < 8; ++q)
            if (idx * 8 + q < n) r[idx * 8 + q] = __float2bfloat16_rn(f[q]);
    }
}

template <int kVecs>  // 16-byte vectors per lane
__global__ void __launch_bounds__(256) softmax_fwd_vec_kernel(__nv_bfloat16* __restrict__ s, int64_t rows, int n,
                                                              int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    __nv_bfloat16* r = s + row * ld;
    const int nvec = (n + 7) / 8;
    const float sl2 = scale * 1.4426950408889634f;
    float v[kVecs][8];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
        const int idx = lane + i * 32;
        if (idx < nvec) {
            load_scores8(r, idx, n, sl2, v[i]);
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) v[i][q] = -INFINITY;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) mx = fmaxf(mx, v[i][q]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            v[i][q] = exp2f(v[i][q] - mx);
            sum += v[i][q];
        }
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
        const int idx = lane + i * 32;
        if (idx < nvec) {
#pragma unroll
            for (int q = 0; q < 8; ++q) v[i][q] *= inv;
            store_row8(r, idx, n, v[i]);
        }
    }
}

__global__ void __launch_bounds__(256) softmax_fwd_long_kernel(__nv_bfloat16* __restrict__ s, int64_t rows, int n,
                                                               int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    __nv_bfloat16* r = s + row * ld;
    const int nvec = (n + 7) / 8;
    const float sl2 = scale * 1.4426950408889634f;
    // pass 1: this lane's running max and sum of exp2(x - max), rescaled whenever the max grows
    float mx = -INFINITY, sum = 0.f;
    for (int idx = lane; idx < nvec; idx += 32) {
        float f[8];
        load_scores8(r, idx, n, sl2, f);
        float vm = f[0];
#pragma unroll
        for (int q = 1; q < 8; ++q) vm = fmaxf(vm, f[q]);
        if (vm > mx) {
            sum *= exp2f(mx - vm);
            mx = vm;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) sum += exp2f(f[q] - mx);
    }
    const float row_max = warp_max(mx);
    sum = warp_sum(mx == -INFINITY ? 0.f : sum * exp2f(mx - row_max));
    const float inv = 1.0f / sum;
    // pass 2: normalised write
    for (int idx = lane; idx < nvec; idx += 32) {
        float f[8];
        load_scores8(r, idx, n, sl2, f);
#pragma unroll
        for (int q = 0; q < 8; ++q) f[q] = exp2f(f[q] - row_max) * inv;
        store_row8(r, idx, n, f);
    }
}

// dS = scale * P * (dP - sum_j dP_j P_j), in place on dP; P and dP stay packed in registers.
template <int kVecs>
__global__ void __launch_bounds__(256) softmax_bwd_vec_kernel(__nv_bfloat16* __restrict__ dp,
                                                              const __nv_bfloat16* __restrict__ p, int64_t rows, int n,
                                                              int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    __nv_bfloat16* dr = dp + row * ld;
    const __nv_bfloat16* pr = p + row * ld;
    const int nvec = (n + 7) / 8;
    uint4 pw[kVecs], dw[kVecs];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
        const int idx = lane + i * 32;
        pw[i] = dw[i] = make_uint4(0, 0, 0, 0);
        if (idx < nvec) {
            pw[i] = reinterpret_cast<const uint4*>(pr)[idx];
            dw[i] = reinterpret_cast<const uint4*>(dr)[idx];
            float pf[8], df[8];
            unpack8(pw[i], pf);
            unpack8(dw[i], df);
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (idx * 8 + q < n) dot += pf[q] * df[q];
        }
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int i = 0; i < kVecs; ++i) {
        const int idx = lane + i * 32;
        if (idx < nvec) {
            float pf[8], df[8];
            unpack8(pw[i], pf);
            unpack8(dw[i], df);
#pragma unroll
            for (int q = 0; q < 8; ++q) df[q] = scale * pf[q] * (df[q] - dot);
            store_row8(dr, idx, n, df);
        }
    }
}

__global__ void __launch_bounds__(256) softmax_bwd_long_kernel(__nv_bfloat16* __restrict__ dp,
                                                               const __nv_bfloat16* __restrict__ p, int64_t rows,
                                                               int n, int64_t ld, float scale) {
    const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    const int lane = threadIdx.x % 32;
    __nv_bfloat16* dr = dp + row * ld;
    const __nv_bfloat16* pr = p + row * ld;
    const int nvec = (n + 7) / 8;
    float dot = 0.f;
    for (int idx = lane; idx < nvec; idx += 32) {
        float pf[8], df[8];
        load_masked8(pr, idx, n, pf);
        load_masked8(dr, idx, n, df);
#pragma unroll
        for (int q = 0; q < 8; ++q) dot += pf[q] * df[q];
    }
    dot = warp_sum(dot);
    for (int idx = lane; idx < nvec; idx += 32) {
        float pf[8], df[8];
        load_masked8(pr, idx, n, pf);
        load_masked8(dr, idx, n, df);
#pragma unroll
        for (int q = 0; q < 8; ++q) df[q] = scale * pf[q] * (df[q] - dot);
        store_row8(dr, idx, n, df);
    }
}

// ------------------------------------------------------------------------------------------------
// Cross entropy against a mixed, smoothed target (timm mixup_target + SoftTargetCrossEntropy):
//   t_c = off + w1 * [c == y_b] + w2 * [c == y_{B-1-b}],  w1 = (on - off) * lam,  w2 = (on - off) * (1 - lam)
//   loss += mean_b( logsumexp(logits_b) - off * sum_c logits_bc - w1 * logits_b[y_b] - w2 * logits_b[y_{B-1-b}] )
//   dlogits = (softmax - t) / B
// The hard call (w1 = 1, w2 = 0, off = 0) computes exactly the plain cross-entropy expressions.  One CTA per row.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cross_entropy_kernel(const __nv_bfloat16* __restrict__ logits,
                                                            const int64_t* __restrict__ target,
                                                            __nv_bfloat16* __restrict__ dlogits,
                                                            float* __restrict__ loss, int* __restrict__ correct,
                                                            int B, int C, float inv_b, float w1, float w2, float off) {
    __shared__ float red[64];
    __shared__ int red_i[8];
    const int row = blockIdx.x;
    const __nv_bfloat16* lr = logits + static_cast<int64_t>(row) * C;
    float mx = -INFINITY;
    int arg = 0;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float v = __bfloat162float(lr[c]);
        if (v > mx) mx = v, arg = c;
    }
    // block arg-max (first index wins on ties, like torch.argmax)
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (om > mx || (om == mx && oa < arg)) mx = om, arg = oa;
    }
    const int w = threadIdx.x / 32, l = threadIdx.x % 32;
    if (l == 0) red[w] = mx, red_i[w] = arg;
    __syncthreads();
    mx = red[0], arg = red_i[0];
    for (int i = 1; i < blockDim.x / 32; ++i)
        if (red[i] > mx || (red[i] == mx && red_i[i] < arg)) mx = red[i], arg = red_i[i];
    float s = 0.f, sx = 0.f;  // sum of exp, sum of logits (the smoothing term)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float v = __bfloat162float(lr[c]);
        s += __expf(v - mx);
        sx += v;
    }
    block_sum2<256>(s, sx, red);
    const float lse = mx + __logf(s);
    const int tgt = static_cast<int>(target[row]);
    const int tgt2 = w2 != 0.f ? static_cast<int>(target[B - 1 - row]) : tgt;
    if (dlogits != nullptr) {
        __nv_bfloat16* dr = dlogits + static_cast<int64_t>(row) * C;
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const float pr = __expf(__bfloat162float(lr[c]) - lse);
            const float t = (c == tgt ? w1 : 0.f) + (c == tgt2 ? w2 : 0.f) + off;
            dr[c] = __float2bfloat16((pr - t) * inv_b);
        }
    }
    if (threadIdx.x == 0) {
        float picked = w1 * __bfloat162float(lr[tgt]);
        if (w2 != 0.f) picked += w2 * __bfloat162float(lr[tgt2]);
        if (off != 0.f) picked += off * sx;
        atomicAdd(loss, (lse - picked) * inv_b);
        if (correct != nullptr && arg == tgt) atomicAdd(correct, 1);
    }
}

// ------------------------------------------------------------------------------------------------
// Patch im2col: images [B, 3, S, S] (fp32 or bf16) -> cols [B * (S/P)^2, Kpad] bf16 with
// k = c * P * P + py * P + px (the Conv2d weight's flattening order); columns >= 3 P^2 are zero.
// MIX (timm Mixup, mode 'batch', image b paired with image B-1-b):
//   0  no mixing;
//   1  Mixup:  x_b * lam + x_{B-1-b} * mlam in fp32, each product and the sum rounded once (no FMA contraction), which
//      is what the fp32 PyTorch expression x.mul_(lam).add_(x.flip(0).mul_(1 - lam)) computes;
//   2  CutMix: pixels in [yl, yh) x [xl, xh) come from image B-1-b, all others from image b.
// ------------------------------------------------------------------------------------------------
template <typename T, int MIX>
__global__ void im2col_kernel(const T* __restrict__ img, __nv_bfloat16* __restrict__ cols, int B, int S, int P,
                              int Kpad, Im2colMix mix) {
    const int G = S / P;
    const int64_t total = static_cast<int64_t>(B) * G * G * Kpad;
    const int K = 3 * P * P;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % Kpad);
        const int64_t patch = i / Kpad;
        float v = 0.f;
        if (k < K) v = im2col_pixel<T, MIX>(img, B, S, P, G, patch, k, mix);
        cols[i] = __float2bfloat16(v);
    }
}

// ------------------------------------------------------------------------------------------------
// Column sums of a [rows, C] bf16 matrix into fp32 (bias gradients that are not fused elsewhere).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out,
                                                     int64_t rows, int C, int rows_per_cta) {
    // blockIdx.x: 8-column vector group of 256 threads' worth (256 * 8 columns), blockIdx.y: row slab
    const int vec = blockIdx.x * blockDim.x + threadIdx.x;
    if (vec * 8 >= C) return;
    const int64_t r0 = static_cast<int64_t>(blockIdx.y) * rows_per_cta;
    const int64_t r1 = min(rows, r0 + rows_per_cta);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int64_t r = r0; r < r1; ++r) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(x + r * C + vec * 8), f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) atomicAdd(out + vec * 8 + q, acc[q]);
}

// ------------------------------------------------------------------------------------------------
// Sum of squares (fp32 or bf16 input) -> atomicAdd into one float. Used for the global grad norm.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) sumsq_kernel(const T* __restrict__ x, int64_t n, float* __restrict__ out) {
    __shared__ float red[64];
    float s = 0.f, dummy = 0.f;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float v = static_cast<float>(x[i]);
        s += v * v;
    }
    block_sum2<256>(s, dummy, red);
    if (threadIdx.x == 0) atomicAdd(out, s);
}

// ------------------------------------------------------------------------------------------------
// Fused sharded AdamW.  One pass over the shard:
//   g   = grad * clip_coef (device scalar; 1.0 when clipping is off)
//   m,v = Adam moments (fp32)
//   w   = w * (1 - lr * wd) - lr * mhat / (sqrt(vhat) + eps)          (decoupled weight decay)
// The fp32 master weight is stored *split*: `hi` is the round-to-nearest bf16 value (this is the
// tensor the next all-gather ships and the GEMMs consume), `lo` is the signed 16-bit remainder so that
// (hi << 16) + lo reproduces the fp32 bits exactly.  No separate bf16 copy, no extra cast pass.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_grad4(const float* g, int64_t i, float (&out)[4]) {
    const float4 v = *reinterpret_cast<const float4*>(g + i);
    out[0] = v.x, out[1] = v.y, out[2] = v.z, out[3] = v.w;
}
__device__ __forceinline__ void load_grad4(const __nv_bfloat16* g, int64_t i, float (&out)[4]) {
    const uint2 v = *reinterpret_cast<const uint2*>(g + i);
    out[0] = bf16_lo(v.x), out[1] = bf16_hi(v.x), out[2] = bf16_lo(v.y), out[3] = bf16_hi(v.y);
}

// Split-fp32 helpers shared by the AdamW update and its EMA: (hi << 16) + lo are the fp32 bits, hi rounded half-up.
__device__ __forceinline__ float merge_split(uint32_t h, uint32_t l) {
    return __int_as_float(static_cast<int32_t>(h << 16) + static_cast<int32_t>(static_cast<int16_t>(l)));
}
__device__ __forceinline__ void split_bits(float w, uint32_t& h_out, uint32_t& l_out) {
    const int32_t nb = __float_as_int(w);
    const int32_t rounded = nb + 0x8000;  // round-half-up: keeps lo in [-32768, 32767] (see split_fp32)
    const int32_t h = rounded >> 16;
    h_out = static_cast<uint32_t>(h) & 0xFFFFu;
    l_out = static_cast<uint32_t>(nb - (h << 16)) & 0xFFFFu;
}

// 4 elements per thread: 8 B (hi) + 8 B (lo) + 16 B (m) + 16 B (v) + 8/16 B (grad) vector accesses.
// EMA (model EMA, timm ModelEmaV2): the moving average of the weights is kept in the master's own split form,
// ema_hi (bf16) + ema_lo (int16), and updated from the new fp32 w while it is still in registers:
//   ema = fmaf(d, ema, (1 - d) * w)        (1 - d formed in fp32, so d = 0 gives ema == w bitwise)
// 8 more bytes per element (ema_hi + ema_lo, read and written); hi / lo / m / v are computed exactly as without it.
// GROUPED (parameter groups, see parallel/param_groups.py): every 64-element chunk i >> 6 of the shard belongs to group
// groups[i >> 6], whose row of group_hyper is (lr_scale, wd).  A 4-element vector never crosses a chunk, so each reads
// its group once and uses lr * lr_scale and 1 - lr * lr_scale * wd, formed in fp32, in place of lr and 1 - lr * wd.
// One byte of traffic per 64 elements; the arithmetic is otherwise the ungrouped kernel's.
template <typename GradT, bool EMA, bool GROUPED = false>
__device__ __forceinline__ void adamw_split_body(uint16_t* __restrict__ hi, int16_t* __restrict__ lo,
                                                 float* __restrict__ m, float* __restrict__ v,
                                                 const GradT* __restrict__ grad, int64_t n,
                                                 const float* __restrict__ clip_coef, float lr, float beta1, float beta2,
                                                 float eps, float wd, float bc1, float bc2,
                                                 const float* __restrict__ hyper, uint16_t* __restrict__ ema_hi,
                                                 int16_t* __restrict__ ema_lo, float ema_decay,
                                                 const uint8_t* __restrict__ groups = nullptr,
                                                 const float* __restrict__ group_hyper = nullptr) {
    const float coef = clip_coef != nullptr ? *clip_coef : 1.0f;
    if (hyper != nullptr) {  // lr and step live on the device so the launch can sit inside a CUDA graph
        lr = hyper[0];
        // 1 - beta^t as -expm1(t * log1p(beta - 1)) (beta - 1 is exact): --use_fast_math turns powf into
        // ex2.approx(t * lg2.approx(beta)), whose ~1e-7 absolute error in lg2(beta2) is a ~1e-4 relative error in
        // 1 - beta2^t at small t, i.e. a 5e-5 error in every update of the first steps
        bc1 = -expm1f(hyper[1] * log1pf(beta1 - 1.f));
        bc2 = -expm1f(hyper[1] * log1pf(beta2 - 1.f));
    }
    const float inv_bc1 = 1.f / bc1, inv_bc2 = 1.f / bc2, decay = 1.f - lr * wd;
    const float ema_keep = 1.f - ema_decay;
    const int64_t n4 = n / 4;
    for (int64_t q = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; q < n4;
         q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int64_t i = q * 4;
        const uint2 hv = *reinterpret_cast<const uint2*>(hi + i);
        const uint2 lv = *reinterpret_cast<const uint2*>(lo + i);
        float4 mv = *reinterpret_cast<const float4*>(m + i);
        float4 vv = *reinterpret_cast<const float4*>(v + i);
        float g[4];
        load_grad4(grad, i, g);
        uint2 ehv, elv;
        if constexpr (EMA) {
            ehv = *reinterpret_cast<const uint2*>(ema_hi + i);
            elv = *reinterpret_cast<const uint2*>(ema_lo + i);
        }
        const uint32_t hw[4] = {hv.x & 0xFFFFu, hv.x >> 16, hv.y & 0xFFFFu, hv.y >> 16};
        const uint32_t lw[4] = {lv.x & 0xFFFFu, lv.x >> 16, lv.y & 0xFFFFu, lv.y >> 16};
        float mm[4] = {mv.x, mv.y, mv.z, mv.w}, vq[4] = {vv.x, vv.y, vv.z, vv.w};
        uint32_t ho[4], lo_o[4], eho[4], elo[4];
        float lr_q = lr, decay_q = decay;
        if constexpr (GROUPED) {
            const int grp = groups[i >> 6];
            lr_q = lr * __ldg(group_hyper + 2 * grp);
            decay_q = 1.f - lr_q * __ldg(group_hyper + 2 * grp + 1);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int32_t bits = static_cast<int32_t>(hw[k] << 16) + static_cast<int32_t>(static_cast<int16_t>(lw[k]));
            float w = __int_as_float(bits);
            const float gk = g[k] * coef;
            mm[k] = beta1 * mm[k] + (1.f - beta1) * gk;
            vq[k] = beta2 * vq[k] + (1.f - beta2) * gk * gk;
            w = w * decay_q - lr_q * (mm[k] * inv_bc1) / (sqrtf(vq[k] * inv_bc2) + eps);
            const int32_t nb = __float_as_int(w);
            const int32_t rounded = nb + 0x8000;  // round-half-up: keeps lo in [-32768, 32767] (see split_fp32)
            const int32_t h = rounded >> 16;
            ho[k] = static_cast<uint32_t>(h) & 0xFFFFu;
            lo_o[k] = static_cast<uint32_t>(nb - (h << 16)) & 0xFFFFu;
            if constexpr (EMA) {
                const uint32_t sh = k & 1 ? 16 : 0;
                const float e = merge_split(((k < 2 ? ehv.x : ehv.y) >> sh) & 0xFFFFu,
                                            ((k < 2 ? elv.x : elv.y) >> sh) & 0xFFFFu);
                split_bits(fmaf(ema_decay, e, ema_keep * w), eho[k], elo[k]);
            }
        }
        *reinterpret_cast<uint2*>(hi + i) = make_uint2(ho[0] | (ho[1] << 16), ho[2] | (ho[3] << 16));
        *reinterpret_cast<uint2*>(lo + i) = make_uint2(lo_o[0] | (lo_o[1] << 16), lo_o[2] | (lo_o[3] << 16));
        *reinterpret_cast<float4*>(m + i) = make_float4(mm[0], mm[1], mm[2], mm[3]);
        *reinterpret_cast<float4*>(v + i) = make_float4(vq[0], vq[1], vq[2], vq[3]);
        if constexpr (EMA) {
            *reinterpret_cast<uint2*>(ema_hi + i) = make_uint2(eho[0] | (eho[1] << 16), eho[2] | (eho[3] << 16));
            *reinterpret_cast<uint2*>(ema_lo + i) = make_uint2(elo[0] | (elo[1] << 16), elo[2] | (elo[3] << 16));
        }
    }
    // scalar tail (n not a multiple of 4; never taken by the grouped kernels, whose n is a multiple of 64)
    if constexpr (GROUPED) return;
    for (int64_t i = n4 * 4 + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t bits = (static_cast<int32_t>(hi[i]) << 16) + static_cast<int32_t>(lo[i]);
        float w = __int_as_float(bits);
        const float gk = static_cast<float>(grad[i]) * coef;
        const float mi = beta1 * m[i] + (1.f - beta1) * gk;
        const float vi = beta2 * v[i] + (1.f - beta2) * gk * gk;
        m[i] = mi;
        v[i] = vi;
        w = w * decay - lr * (mi * inv_bc1) / (sqrtf(vi * inv_bc2) + eps);
        const int32_t nb = __float_as_int(w);
        const int32_t rounded = nb + 0x8000;
        const int32_t h = rounded >> 16;
        hi[i] = static_cast<uint16_t>(h & 0xFFFF);
        lo[i] = static_cast<int16_t>(nb - (h << 16));
        if constexpr (EMA) {
            const float e = merge_split(ema_hi[i], static_cast<uint16_t>(ema_lo[i]));
            uint32_t eh, el;
            split_bits(fmaf(ema_decay, e, ema_keep * w), eh, el);
            ema_hi[i] = static_cast<uint16_t>(eh);
            ema_lo[i] = static_cast<int16_t>(static_cast<uint16_t>(el));
        }
    }
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_split_kernel(uint16_t* __restrict__ hi, int16_t* __restrict__ lo,
                                                          float* __restrict__ m, float* __restrict__ v,
                                                          const GradT* __restrict__ grad, int64_t n,
                                                          const float* __restrict__ clip_coef, float lr, float beta1,
                                                          float beta2, float eps, float wd, float bc1, float bc2,
                                                          const float* __restrict__ hyper) {
    adamw_split_body<GradT, false>(hi, lo, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2, hyper,
                                   nullptr, nullptr, 0.f);
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_split_ema_kernel(uint16_t* __restrict__ hi, int16_t* __restrict__ lo,
                                                              float* __restrict__ m, float* __restrict__ v,
                                                              const GradT* __restrict__ grad, int64_t n,
                                                              const float* __restrict__ clip_coef, float lr,
                                                              float beta1, float beta2, float eps, float wd, float bc1,
                                                              float bc2, const float* __restrict__ hyper,
                                                              uint16_t* __restrict__ ema_hi,
                                                              int16_t* __restrict__ ema_lo, float ema_decay) {
    adamw_split_body<GradT, true>(hi, lo, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2, hyper,
                                  ema_hi, ema_lo, ema_decay);
}

// Parameter-group variants of the two kernels above (n % 64 == 0).
template <typename GradT>
__global__ void __launch_bounds__(256) adamw_split_grouped_kernel(
    uint16_t* __restrict__ hi, int16_t* __restrict__ lo, float* __restrict__ m, float* __restrict__ v,
    const GradT* __restrict__ grad, int64_t n, const float* __restrict__ clip_coef, float lr, float beta1, float beta2,
    float eps, float bc1, float bc2, const float* __restrict__ hyper, const uint8_t* __restrict__ groups,
    const float* __restrict__ group_hyper) {
    adamw_split_body<GradT, false, true>(hi, lo, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, 0.f, bc1, bc2, hyper,
                                         nullptr, nullptr, 0.f, groups, group_hyper);
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_split_ema_grouped_kernel(
    uint16_t* __restrict__ hi, int16_t* __restrict__ lo, float* __restrict__ m, float* __restrict__ v,
    const GradT* __restrict__ grad, int64_t n, const float* __restrict__ clip_coef, float lr, float beta1, float beta2,
    float eps, float bc1, float bc2, const float* __restrict__ hyper, uint16_t* __restrict__ ema_hi,
    int16_t* __restrict__ ema_lo, float ema_decay, const uint8_t* __restrict__ groups,
    const float* __restrict__ group_hyper) {
    adamw_split_body<GradT, true, true>(hi, lo, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, 0.f, bc1, bc2, hyper,
                                        ema_hi, ema_lo, ema_decay, groups, group_hyper);
}

// Plain fp32-master variant (used when the compute dtype is fp32); the EMA is a plain fp32 shard here.
template <typename GradT, bool EMA, bool GROUPED = false>
__device__ __forceinline__ void adamw_fp32_body(float* __restrict__ w, float* __restrict__ m, float* __restrict__ v,
                                                const GradT* __restrict__ grad, int64_t n,
                                                const float* __restrict__ clip_coef, float lr, float beta1, float beta2,
                                                float eps, float wd, float bc1, float bc2, float* __restrict__ ema,
                                                float ema_decay, const uint8_t* __restrict__ groups = nullptr,
                                                const float* __restrict__ group_hyper = nullptr) {
    const float coef = clip_coef != nullptr ? *clip_coef : 1.0f;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const float g = static_cast<float>(grad[i]) * coef;
        const float mi = beta1 * m[i] + (1.f - beta1) * g;
        const float vi = beta2 * v[i] + (1.f - beta2) * g * g;
        m[i] = mi;
        v[i] = vi;
        float lr_i = lr, wd_i = wd;
        if constexpr (GROUPED) {
            const int grp = groups[i >> 6];
            lr_i = lr * __ldg(group_hyper + 2 * grp);
            wd_i = __ldg(group_hyper + 2 * grp + 1);
        }
        const float wi = w[i] * (1.f - lr_i * wd_i) - lr_i * (mi / bc1) / (sqrtf(vi / bc2) + eps);
        w[i] = wi;
        if constexpr (EMA) ema[i] = fmaf(ema_decay, ema[i], (1.f - ema_decay) * wi);
    }
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_fp32_kernel(float* __restrict__ w, float* __restrict__ m,
                                                         float* __restrict__ v, const GradT* __restrict__ grad,
                                                         int64_t n, const float* __restrict__ clip_coef, float lr,
                                                         float beta1, float beta2, float eps, float wd, float bc1,
                                                         float bc2) {
    adamw_fp32_body<GradT, false>(w, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2, nullptr, 0.f);
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_fp32_ema_kernel(float* __restrict__ w, float* __restrict__ m,
                                                             float* __restrict__ v, const GradT* __restrict__ grad,
                                                             int64_t n, const float* __restrict__ clip_coef, float lr,
                                                             float beta1, float beta2, float eps, float wd, float bc1,
                                                             float bc2, float* __restrict__ ema, float ema_decay) {
    adamw_fp32_body<GradT, true>(w, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2, ema, ema_decay);
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_fp32_grouped_kernel(
    float* __restrict__ w, float* __restrict__ m, float* __restrict__ v, const GradT* __restrict__ grad, int64_t n,
    const float* __restrict__ clip_coef, float lr, float beta1, float beta2, float eps, float bc1, float bc2,
    const uint8_t* __restrict__ groups, const float* __restrict__ group_hyper) {
    adamw_fp32_body<GradT, false, true>(w, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, 0.f, bc1, bc2, nullptr, 0.f,
                                        groups, group_hyper);
}

template <typename GradT>
__global__ void __launch_bounds__(256) adamw_fp32_ema_grouped_kernel(
    float* __restrict__ w, float* __restrict__ m, float* __restrict__ v, const GradT* __restrict__ grad, int64_t n,
    const float* __restrict__ clip_coef, float lr, float beta1, float beta2, float eps, float bc1, float bc2,
    float* __restrict__ ema, float ema_decay, const uint8_t* __restrict__ groups, const float* __restrict__ group_hyper) {
    adamw_fp32_body<GradT, true, true>(w, m, v, grad, n, clip_coef, lr, beta1, beta2, eps, 0.f, bc1, bc2, ema, ema_decay,
                                       groups, group_hyper);
}

// Split an fp32 tensor into (hi bf16, lo int16) and back.
__global__ void split_fp32_kernel(const float* __restrict__ w, uint16_t* __restrict__ hi, int16_t* __restrict__ lo,
                                  int64_t n) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int32_t nb = __float_as_int(w[i]);
        const int32_t rounded = nb + 0x8000;
        const int32_t h = rounded >> 16;
        hi[i] = static_cast<uint16_t>(h & 0xFFFF);
        lo[i] = static_cast<int16_t>(nb - (h << 16));
    }
}
__global__ void merge_fp32_kernel(const uint16_t* __restrict__ hi, const int16_t* __restrict__ lo,
                                  float* __restrict__ w, int64_t n) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        w[i] = __int_as_float((static_cast<int32_t>(hi[i]) << 16) + static_cast<int32_t>(lo[i]));
    }
}

// clip_coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)); also publishes the norm.
__global__ void clip_coef_kernel(const float* __restrict__ sumsq, float max_norm, float* __restrict__ coef,
                                 float* __restrict__ norm_out) {
    const float norm = sqrtf(*sumsq);
    if (norm_out != nullptr) *norm_out = norm;
    *coef = fminf(1.0f, max_norm / (norm + 1e-6f));
}

inline void check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}

}  // namespace

#define LN_DISPATCH(CH, KERNEL, ...)                                       \
    switch (CH) {                                                          \
        case 1: KERNEL<1><<<grid, kLnThreads, 0, stream>>>(__VA_ARGS__); break; \
        case 2: KERNEL<2><<<grid, kLnThreads, 0, stream>>>(__VA_ARGS__); break; \
        case 3: KERNEL<3><<<grid, kLnThreads, 0, stream>>>(__VA_ARGS__); break; \
        case 4: KERNEL<4><<<grid, kLnThreads, 0, stream>>>(__VA_ARGS__); break; \
        default: throw std::runtime_error("layernorm: width > 8192 not supported"); \
    }

#define LN_SMALL_DISPATCH(KERNEL, SMEM_FLOATS_PER_COL, CTAS_PER_SM, ...)                                                  \
    {                                                                                   \
        const int nv = D / 8;                                                           \
        const int tpr = nv <= 32 ? 32 : (nv <= 64 ? 64 : (nv <= 128 ? 128 : 256));      \
        const int rows_per = kLnThreads / tpr;                                          \
        const int grid = std::min((rows + rows_per - 1) / rows_per, sm_count() * CTAS_PER_SM);    \
        const size_t smem = SMEM_FLOATS_PER_COL * tpr * 8 * sizeof(float);              \
        if (tpr == 32) KERNEL<32><<<grid, kLnThreads, smem, stream>>>(__VA_ARGS__);        \
        else if (tpr == 64) KERNEL<64><<<grid, kLnThreads, smem, stream>>>(__VA_ARGS__);   \
        else if (tpr == 128) KERNEL<128><<<grid, kLnThreads, smem, stream>>>(__VA_ARGS__); \
        else KERNEL<256><<<grid, kLnThreads, smem, stream>>>(__VA_ARGS__);                 \
    }

void layernorm_fwd(const __nv_bfloat16* x, const __nv_bfloat16* gamma, const __nv_bfloat16* beta, __nv_bfloat16* y,
                   float* mean, float* rstd, int rows, int D, float eps, cudaStream_t stream) {
    if (D % 8 != 0) throw std::runtime_error("layernorm: width must be a multiple of 8");
    static const bool ln_small = getenv("B200_LN_SMALL") == nullptr || atoi(getenv("B200_LN_SMALL")) != 0;
    if (D <= 2048 && ln_small) {
        LN_SMALL_DISPATCH(ln_fwd_small_kernel, 0, 6, x, gamma, beta, y, mean, rstd, rows, D, eps);
        check_launch("layernorm_fwd_small");
        return;
    }
    const int chunks = (D / 8 + kLnThreads - 1) / kLnThreads;
    const int grid = std::min(rows, sm_count() * 8);
    LN_DISPATCH(chunks, ln_fwd_kernel, x, gamma, beta, y, mean, rstd, rows, D, eps);
    check_launch("layernorm_fwd");
}

template <int kChunks>
void launch_ln_bwd(int grid, size_t smem, cudaStream_t stream, const __nv_bfloat16* dy, const __nv_bfloat16* x,
                   const __nv_bfloat16* gamma, const float* mean, const float* rstd, const __nv_bfloat16* dres,
                   __nv_bfloat16* dx, float* dgamma, float* dbeta, float* dxsum, int rows, int D) {
    static size_t configured = 0;
    if (smem > configured) {
        cudaFuncSetAttribute(ln_bwd_kernel<kChunks>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        configured = smem;
    }
    ln_bwd_kernel<kChunks><<<grid, kLnThreads, smem, stream>>>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum,
                                                             rows, D);
}

void layernorm_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                   const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                   float* dxsum, int rows, int D, cudaStream_t stream) {
    if (D % 8 != 0) throw std::runtime_error("layernorm: width must be a multiple of 8");
    static const bool ln_small = getenv("B200_LN_SMALL") == nullptr || atoi(getenv("B200_LN_SMALL")) != 0;
    if (D <= 2048 && ln_small) {
        LN_SMALL_DISPATCH(ln_bwd_small_kernel, 3, 4, dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D);
        check_launch("layernorm_bwd_small");
        return;
    }
    static const bool ln_stream = getenv("B200_LN_STREAM") == nullptr || atoi(getenv("B200_LN_STREAM")) != 0;
    if (ln_stream && layernorm_bwd_stream_supported(D) && rows >= sm_count()) {
        layernorm_bwd_stream(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
        return;
    }
    const int chunks = (D / 8 + kLnThreads - 1) / kLnThreads;
    const size_t smem = static_cast<size_t>(dxsum != nullptr ? 3 : 2) * D * sizeof(float);
    const int per_sm = std::max<int>(1, std::min<int>(3, static_cast<int>((200 * 1024) / std::max<size_t>(smem, 1))));
    const int grid = std::min(rows, sm_count() * per_sm);
    switch (chunks) {
        case 1: launch_ln_bwd<1>(grid, smem, stream, dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D); break;
        case 2: launch_ln_bwd<2>(grid, smem, stream, dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D); break;
        case 3: launch_ln_bwd<3>(grid, smem, stream, dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D); break;
        case 4: launch_ln_bwd<4>(grid, smem, stream, dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D); break;
        default: throw std::runtime_error("layernorm: width > 8192 not supported");
    }
    check_launch("layernorm_bwd");
}

#define SM_DISPATCH(KERNEL, ...)                                                                   \
    if (pairs_per_lane <= 2) KERNEL<2><<<grid, 256, 0, stream>>>(__VA_ARGS__);                     \
    else if (pairs_per_lane <= 4) KERNEL<4><<<grid, 256, 0, stream>>>(__VA_ARGS__);                \
    else if (pairs_per_lane <= 9) KERNEL<9><<<grid, 256, 0, stream>>>(__VA_ARGS__);                \
    else KERNEL<16><<<grid, 256, 0, stream>>>(__VA_ARGS__);

// The bf16x2 pair kernels take even n <= 1024; the vector kernels take every other row length.
static bool softmax_pairs(int n) { return n % 2 == 0 && n <= 1024; }

static void check_softmax_args(const void* a, const void* b, int n, int64_t ld) {
    if (n < 1) throw std::runtime_error("softmax: row length n must be >= 1");
    if (ld < n) throw std::runtime_error("softmax: ld must be >= row length n");
    if (softmax_pairs(n)) {
        if (ld % 2 != 0) throw std::runtime_error("softmax: ld must be even");
    } else {
        if (ld % 8 != 0) throw std::runtime_error("softmax: ld must be a multiple of 8 for odd n or n > 1024");
        if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) % 16 != 0)
            throw std::runtime_error("softmax: buffers must be 16-byte aligned for odd n or n > 1024");
    }
}

#define SM_VEC_DISPATCH(KERNEL, LONG_KERNEL, ...)                                                  \
    if (vecs_per_lane <= 1) KERNEL<1><<<grid, 256, 0, stream>>>(__VA_ARGS__);                      \
    else if (vecs_per_lane <= 2) KERNEL<2><<<grid, 256, 0, stream>>>(__VA_ARGS__);                 \
    else if (vecs_per_lane <= 4) KERNEL<4><<<grid, 256, 0, stream>>>(__VA_ARGS__);                 \
    else if (n <= kSoftmaxRegMaxN) KERNEL<8><<<grid, 256, 0, stream>>>(__VA_ARGS__);               \
    else LONG_KERNEL<<<grid, 256, 0, stream>>>(__VA_ARGS__);

void softmax_fwd(__nv_bfloat16* s, int64_t rows, int n, int64_t ld, float scale, cudaStream_t stream) {
    check_softmax_args(s, s, n, ld);
    if (rows == 0) return;
    const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
    if (softmax_pairs(n)) {
        const int pairs_per_lane = (n / 2 + 31) / 32;
        SM_DISPATCH(softmax_fwd_kernel, s, rows, n, ld, scale);
    } else {
        const int vecs_per_lane = ((n + 7) / 8 + 31) / 32;
        SM_VEC_DISPATCH(softmax_fwd_vec_kernel, softmax_fwd_long_kernel, s, rows, n, ld, scale);
    }
    check_launch("softmax_fwd");
}

void softmax_bwd(__nv_bfloat16* dp, const __nv_bfloat16* p, int64_t rows, int n, int64_t ld, float scale,
                 cudaStream_t stream) {
    check_softmax_args(dp, p, n, ld);
    if (rows == 0) return;
    const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
    if (softmax_pairs(n)) {
        const int pairs_per_lane = (n / 2 + 31) / 32;
        SM_DISPATCH(softmax_bwd_kernel, dp, p, rows, n, ld, scale);
    } else {
        const int vecs_per_lane = ((n + 7) / 8 + 31) / 32;
        SM_VEC_DISPATCH(softmax_bwd_vec_kernel, softmax_bwd_long_kernel, dp, p, rows, n, ld, scale);
    }
    check_launch("softmax_bwd");
}

void cross_entropy(const __nv_bfloat16* logits, const int64_t* target, __nv_bfloat16* dlogits, float* loss,
                   int* correct, int B, int C, cudaStream_t stream, double lam, double smoothing) {
    // target weights in double, rounded once: lam = 1, smoothing = 0 gives exactly w1 = 1, w2 = 0, off = 0
    const double off = smoothing / C, on = 1.0 - smoothing + off;
    const float w1 = static_cast<float>((on - off) * lam), w2 = static_cast<float>((on - off) * (1.0 - lam));
    if (w2 != 0.f && B % 2 != 0) throw std::runtime_error("cross_entropy: mixed targets need an even batch");
    cross_entropy_kernel<<<B, 256, 0, stream>>>(logits, target, dlogits, loss, correct, B, C, 1.0f / B, w1, w2,
                                                static_cast<float>(off));
    check_launch("cross_entropy");
}

template <typename T>
static void im2col_launch(const T* img, __nv_bfloat16* cols, int B, int S, int P, int Kpad, const Im2colMix& mix,
                          cudaStream_t stream) {
    const int grid = sm_count() * 8;
    if (mix.mode == 0)
        im2col_kernel<T, 0><<<grid, 256, 0, stream>>>(img, cols, B, S, P, Kpad, mix);
    else if (mix.mode == 1)
        im2col_kernel<T, 1><<<grid, 256, 0, stream>>>(img, cols, B, S, P, Kpad, mix);
    else
        im2col_kernel<T, 2><<<grid, 256, 0, stream>>>(img, cols, B, S, P, Kpad, mix);
}

void im2col(const void* img, bool img_is_bf16, __nv_bfloat16* cols, int B, int S, int P, int Kpad,
            cudaStream_t stream, const Im2colMix& mix) {
    if (mix.mode < 0 || mix.mode > 2) throw std::runtime_error("im2col: mix mode must be 0, 1 or 2");
    if (mix.mode != 0 && B % 2 != 0) throw std::runtime_error("im2col: batch mixing needs an even batch");
    if (mix.mode == 2 && !(0 <= mix.yl && mix.yl <= mix.yh && mix.yh <= S && 0 <= mix.xl && mix.xl <= mix.xh &&
                           mix.xh <= S))
        throw std::runtime_error("im2col: the CutMix box must lie inside the image");
    if (img_is_bf16)
        im2col_launch(static_cast<const __nv_bfloat16*>(img), cols, B, S, P, Kpad, mix, stream);
    else
        im2col_launch(static_cast<const float*>(img), cols, B, S, P, Kpad, mix, stream);
    check_launch("im2col");
}

void gelu_fwd(const __nv_bfloat16* u, __nv_bfloat16* g, int64_t n, cudaStream_t stream) {
    if (n % 8 != 0) throw std::runtime_error("gelu: element count must be a multiple of 8");
    const int grid = static_cast<int>(std::min<int64_t>((n / 8 + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    gelu_fwd_kernel<<<grid, 256, 0, stream>>>(u, g, n / 8);
    check_launch("gelu_fwd");
}

void dgelu_mul(const __nv_bfloat16* dg, const __nv_bfloat16* u, __nv_bfloat16* du, int64_t n, cudaStream_t stream) {
    if (n % 8 != 0) throw std::runtime_error("dgelu: element count must be a multiple of 8");
    const int grid = static_cast<int>(std::min<int64_t>((n / 8 + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    dgelu_mul_kernel<<<grid, 256, 0, stream>>>(dg, u, du, n / 8);
    check_launch("dgelu_mul");
}

void swiglu_fwd(const __nv_bfloat16* u, __nv_bfloat16* g, int64_t M, int64_t hidden, cudaStream_t stream) {
    if (M < 0 || hidden < 0 || hidden % 16 != 0)
        throw std::runtime_error("swiglu_fwd: the packed width Hd must be a multiple of 16 (16-byte halves)");
    if ((reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(g)) & 15)
        throw std::runtime_error("swiglu_fwd: u and g must be 16-byte aligned");
    const int hvec = static_cast<int>(hidden / 16);
    if (M == 0 || hvec == 0) return;
    const int gx = std::min((hvec + 255) / 256, 64);
    const int64_t gy = std::min<int64_t>(std::min<int64_t>(M, std::max(1, sm_count() * 16 / gx)), 65535);
    const dim3 grid(gx, static_cast<unsigned>(gy));
    swiglu_fwd_kernel<<<grid, 256, 0, stream>>>(u, g, M, hvec);
    check_launch("swiglu_fwd");
}

void swiglu_bwd(const __nv_bfloat16* dg, const __nv_bfloat16* u, __nv_bfloat16* du, int64_t M, int64_t hidden,
                cudaStream_t stream) {
    if (M < 0 || hidden < 0 || hidden % 16 != 0)
        throw std::runtime_error("swiglu_bwd: the packed width Hd must be a multiple of 16 (16-byte halves)");
    if ((reinterpret_cast<uintptr_t>(dg) | reinterpret_cast<uintptr_t>(u) | reinterpret_cast<uintptr_t>(du)) & 15)
        throw std::runtime_error("swiglu_bwd: dg, u and du must be 16-byte aligned");
    const int hvec = static_cast<int>(hidden / 16);
    if (M == 0 || hvec == 0) return;
    const int gx = std::min((hvec + 255) / 256, 64);
    const int64_t gy = std::min<int64_t>(std::min<int64_t>(M, std::max(1, sm_count() * 16 / gx)), 65535);
    const dim3 grid(gx, static_cast<unsigned>(gy));
    swiglu_bwd_kernel<<<grid, 256, 0, stream>>>(dg, u, du, M, hvec);
    check_launch("swiglu_bwd");
}

void dropout(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, float p, uint64_t key, cudaStream_t stream) {
    if (n % 8 != 0) throw std::runtime_error("dropout: element count must be a multiple of 8");
    if (!(p >= 0.f && p < 1.f)) throw std::runtime_error("dropout: p must be in [0, 1)");
    const int grid = static_cast<int>(std::min<int64_t>((n / 8 + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    const uint32_t thresh = dropout_thresh16(p);
    dropout_kernel<<<grid, 256, 0, stream>>>(x, y, n / 8, static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32),
                                            thresh, dropout_scale(thresh));
    check_launch("dropout");
}

void drop_path_scale(float* scale, int B, int64_t sample_offset, float p, uint64_t key, cudaStream_t stream) {
    if (!(p >= 0.f && p < 1.f)) throw std::runtime_error("drop_path_scale: p must be in [0, 1)");
    if (B < 0 || sample_offset < 0) throw std::runtime_error("drop_path_scale: B and sample_offset must be >= 0");
    if (B == 0) return;
    const uint32_t thresh = dropout_thresh16(p);
    drop_path_scale_kernel<<<(B + 127) / 128, 128, 0, stream>>>(scale, B, sample_offset, static_cast<uint32_t>(key),
                                                                static_cast<uint32_t>(key >> 32), thresh,
                                                                dropout_scale(thresh));
    check_launch("drop_path_scale");
}

void drop_path_bwd(const __nv_bfloat16* dy, const float* scale, __nv_bfloat16* dt, float* colsum, int64_t rows, int C,
                   int N, cudaStream_t stream) {
    if (C % 8 != 0) throw std::runtime_error("drop_path_bwd: width must be a multiple of 8");
    if (N < 1 || rows % N != 0) throw std::runtime_error("drop_path_bwd: rows must be a whole number of N-row samples");
    if ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dt)) & 15)
        throw std::runtime_error("drop_path_bwd: dy and dt must be 16-byte aligned");
    if (rows == 0) return;
    const int gx = (C / 8 + 255) / 256;
    int slabs = std::max(1, (sm_count() * 4) / gx);
    int rows_per = static_cast<int>((rows + slabs - 1) / slabs);
    if (rows_per < 1) rows_per = 1;
    slabs = static_cast<int>((rows + rows_per - 1) / rows_per);
    drop_path_bwd_kernel<<<dim3(gx, slabs), 256, 0, stream>>>(dy, scale, dt, colsum, rows, C, N, rows_per);
    check_launch("drop_path_bwd");
}

void meanpool_fwd(const __nv_bfloat16* xn, __nv_bfloat16* pooled, int B, int N, int D, cudaStream_t stream) {
    if (D % 8 != 0) throw std::runtime_error("meanpool: width must be a multiple of 8");
    dim3 grid((D / 8 + 127) / 128, B);
    meanpool_fwd_kernel<<<grid, 128, 0, stream>>>(xn, pooled, N, D);
    check_launch("meanpool_fwd");
}

void meanpool_bwd(const __nv_bfloat16* dpooled, __nv_bfloat16* dxn, int B, int N, int D, cudaStream_t stream) {
    if (D % 8 != 0) throw std::runtime_error("meanpool: width must be a multiple of 8");
    dim3 grid((D / 8 + 127) / 128, B);
    meanpool_bwd_kernel<<<grid, 128, 0, stream>>>(dpooled, dxn, N, D);
    check_launch("meanpool_bwd");
}

void colsum(const __nv_bfloat16* x, float* out, int64_t rows, int C, cudaStream_t stream) {
    if (C % 8 != 0) throw std::runtime_error("colsum: width must be a multiple of 8");
    const int gx = (C / 8 + 255) / 256;
    int slabs = std::max(1, (sm_count() * 4) / gx);
    int rows_per = static_cast<int>((rows + slabs - 1) / slabs);
    if (rows_per < 1) rows_per = 1;
    slabs = static_cast<int>((rows + rows_per - 1) / rows_per);
    colsum_kernel<<<dim3(gx, slabs), 256, 0, stream>>>(x, out, rows, C, rows_per);
    check_launch("colsum");
}

void sumsq(const void* x, bool is_bf16, int64_t n, float* out, cudaStream_t stream) {
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, sm_count() * 8));
    if (grid == 0) return;
    if (is_bf16)
        sumsq_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), n, out);
    else
        sumsq_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(x), n, out);
    check_launch("sumsq");
}

void adamw_split(uint16_t* hi, int16_t* lo, float* m, float* v, const void* grad, bool grad_is_bf16, int64_t n,
                 const float* clip_coef, float lr, float beta1, float beta2, float eps, float wd, int step,
                 cudaStream_t stream, const float* hyper, uint16_t* ema_hi, int16_t* ema_lo, float ema_decay,
                 const uint8_t* groups, const float* group_hyper) {
    if ((ema_hi == nullptr) != (ema_lo == nullptr))
        throw std::runtime_error("adamw_split: the EMA needs both ema_hi and ema_lo (or neither)");
    if ((groups == nullptr) != (group_hyper == nullptr))
        throw std::runtime_error("adamw_split: the parameter groups need both groups and group_hyper (or neither)");
    if (groups != nullptr && n % 64 != 0) throw std::runtime_error("adamw_split: grouped update needs n % 64 == 0");
    const int grid = static_cast<int>(std::min<int64_t>((n / 4 + 255) / 256 + 1, sm_count() * 16));
    if (grid == 0) return;
    // 1 - beta^t in double: in fp32, 1 - powf(0.999f, 2) keeps only the rounding error of powf (1.5e-5 of 0.002)
    const float bc1 = static_cast<float>(1.0 - std::pow(static_cast<double>(beta1), static_cast<double>(step)));
    const float bc2 = static_cast<float>(1.0 - std::pow(static_cast<double>(beta2), static_cast<double>(step)));
    if (groups != nullptr) {
        if (ema_hi != nullptr && grad_is_bf16)
            adamw_split_ema_grouped_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                hi, lo, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2,
                hyper, ema_hi, ema_lo, ema_decay, groups, group_hyper);
        else if (ema_hi != nullptr)
            adamw_split_ema_grouped_kernel<float><<<grid, 256, 0, stream>>>(
                hi, lo, m, v, static_cast<const float*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, hyper,
                ema_hi, ema_lo, ema_decay, groups, group_hyper);
        else if (grad_is_bf16)
            adamw_split_grouped_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                hi, lo, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2,
                hyper, groups, group_hyper);
        else
            adamw_split_grouped_kernel<float><<<grid, 256, 0, stream>>>(
                hi, lo, m, v, static_cast<const float*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, hyper,
                groups, group_hyper);
    } else if (ema_hi != nullptr) {
        if (grad_is_bf16)
            adamw_split_ema_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                hi, lo, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, wd, bc1,
                bc2, hyper, ema_hi, ema_lo, ema_decay);
        else
            adamw_split_ema_kernel<float><<<grid, 256, 0, stream>>>(hi, lo, m, v, static_cast<const float*>(grad), n,
                                                                   clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2,
                                                                   hyper, ema_hi, ema_lo, ema_decay);
    } else if (grad_is_bf16) {
        adamw_split_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(hi, lo, m, v, static_cast<const __nv_bfloat16*>(grad),
                                                                   n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2,
                                                                   hyper);
    } else {
        adamw_split_kernel<float><<<grid, 256, 0, stream>>>(hi, lo, m, v, static_cast<const float*>(grad), n, clip_coef,
                                                           lr, beta1, beta2, eps, wd, bc1, bc2, hyper);
    }
    check_launch("adamw_split");
}

void adamw_fp32(float* w, float* m, float* v, const void* grad, bool grad_is_bf16, int64_t n, const float* clip_coef,
                float lr, float beta1, float beta2, float eps, float wd, int step, cudaStream_t stream, float* ema,
                float ema_decay, const uint8_t* groups, const float* group_hyper) {
    if ((groups == nullptr) != (group_hyper == nullptr))
        throw std::runtime_error("adamw_fp32: the parameter groups need both groups and group_hyper (or neither)");
    if (groups != nullptr && n % 64 != 0) throw std::runtime_error("adamw_fp32: grouped update needs n % 64 == 0");
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    // 1 - beta^t in double: in fp32, 1 - powf(0.999f, 2) keeps only the rounding error of powf (1.5e-5 of 0.002)
    const float bc1 = static_cast<float>(1.0 - std::pow(static_cast<double>(beta1), static_cast<double>(step)));
    const float bc2 = static_cast<float>(1.0 - std::pow(static_cast<double>(beta2), static_cast<double>(step)));
    if (groups != nullptr) {
        if (ema != nullptr && grad_is_bf16)
            adamw_fp32_ema_grouped_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                w, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, ema,
                ema_decay, groups, group_hyper);
        else if (ema != nullptr)
            adamw_fp32_ema_grouped_kernel<float><<<grid, 256, 0, stream>>>(
                w, m, v, static_cast<const float*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, ema, ema_decay,
                groups, group_hyper);
        else if (grad_is_bf16)
            adamw_fp32_grouped_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                w, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, groups,
                group_hyper);
        else
            adamw_fp32_grouped_kernel<float><<<grid, 256, 0, stream>>>(
                w, m, v, static_cast<const float*>(grad), n, clip_coef, lr, beta1, beta2, eps, bc1, bc2, groups,
                group_hyper);
    } else if (ema != nullptr) {
        if (grad_is_bf16)
            adamw_fp32_ema_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
                w, m, v, static_cast<const __nv_bfloat16*>(grad), n, clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2, ema,
                ema_decay);
        else
            adamw_fp32_ema_kernel<float><<<grid, 256, 0, stream>>>(w, m, v, static_cast<const float*>(grad), n, clip_coef,
                                                                  lr, beta1, beta2, eps, wd, bc1, bc2, ema, ema_decay);
    } else if (grad_is_bf16) {
        adamw_fp32_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(w, m, v, static_cast<const __nv_bfloat16*>(grad), n,
                                                                  clip_coef, lr, beta1, beta2, eps, wd, bc1, bc2);
    } else {
        adamw_fp32_kernel<float><<<grid, 256, 0, stream>>>(w, m, v, static_cast<const float*>(grad), n, clip_coef, lr,
                                                          beta1, beta2, eps, wd, bc1, bc2);
    }
    check_launch("adamw_fp32");
}

void split_fp32(const float* w, uint16_t* hi, int16_t* lo, int64_t n, cudaStream_t stream) {
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    split_fp32_kernel<<<grid, 256, 0, stream>>>(w, hi, lo, n);
    check_launch("split_fp32");
}

void merge_fp32(const uint16_t* hi, const int16_t* lo, float* w, int64_t n, cudaStream_t stream) {
    const int grid = static_cast<int>(std::min<int64_t>((n + 255) / 256, sm_count() * 16));
    if (grid == 0) return;
    merge_fp32_kernel<<<grid, 256, 0, stream>>>(hi, lo, w, n);
    check_launch("merge_fp32");
}

void clip_coef(const float* sumsq_in, float max_norm, float* coef, float* norm_out, cudaStream_t stream) {
    clip_coef_kernel<<<1, 1, 0, stream>>>(sumsq_in, max_norm, coef, norm_out);
    check_launch("clip_coef");
}

}  // namespace b200
