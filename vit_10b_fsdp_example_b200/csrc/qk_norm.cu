// QK normalisation (timm Attention(qk_norm=True), ViT-22B): a LayerNorm over the head dim of every query and key head,
// run on the packed [T, 3D] qkv buffer the qkv GEMM writes and the attention kernels read (D = H * hd).  Row t holds H
// query heads, then H key heads, then H value heads, each hd wide.
//
// A (token, head) row is short (hd = 160 is 20 16-byte vectors), so a group of 8 lanes (16 in the backward for hd > 128)
// owns one head slot j of the row (j < H: query head j, j < 2H: key head j - H, j < 3H: value head, copied by the
// out-of-place forward) and walks a slab of tokens; each lane holds kVpl vectors of the head, and the statistics are
// reduced over the group with shuffles.  A CTA covers 32 (or 16) consecutive head slots of the same tokens, so its loads
// are contiguous runs of heads and, in the backward, each column of the qkv bias gradient is owned by one group per CTA.
// Statistics and gradients are fp32; each bf16 output is rounded once.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "elementwise.h"
#include "ptx.cuh"
#include "rope.cuh"

namespace b200 {

namespace {

constexpr int kQkLanes = 8;                        // lanes per (token, head) row in the forward
constexpr int kQkThreads = 256;
constexpr int kQkGroups = kQkThreads / kQkLanes;   // head slots per forward CTA
constexpr int kQkMaxHd = 256;                      // forward kVpl <= 4: 8 lanes x 4 vectors x 8 columns

__device__ __forceinline__ void qk_unpack8(const uint4& v, float (&f)[8]) {
    f[0] = bf16_lo(v.x), f[1] = bf16_hi(v.x), f[2] = bf16_lo(v.y), f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z), f[5] = bf16_hi(v.z), f[6] = bf16_lo(v.w), f[7] = bf16_hi(v.w);
}
__device__ __forceinline__ uint4 qk_pack8(const float (&f)[8]) {
    uint4 v;
    v.x = pack_bf16x2(f[0], f[1]), v.y = pack_bf16x2(f[2], f[3]);
    v.z = pack_bf16x2(f[4], f[5]), v.w = pack_bf16x2(f[6], f[7]);
    return v;
}

// Sum over the kLanes lanes of a group.  The mask names the group only: a group whose head slot is out of range has left.
template <int kLanes>
__device__ __forceinline__ float group_sum(float v, unsigned mask) {
#pragma unroll
    for (int o = 1; o < kLanes; o <<= 1) v += __shfl_xor_sync(mask, v, o);
    return v;
}
template <int kLanes>
__device__ __forceinline__ unsigned group_mask() {
    return ((1u << kLanes) - 1u) << ((threadIdx.x % 32) & ~(kLanes - 1));
}

// out[:, 0:2D) = LayerNorm_hd of every q / k head; mean / rstd [T, 2, H].  Out of place (slots == 3H) the v heads are
// copied to out as they are; in place (out == qkv, slots == 2H) they are not touched.  qkv / out are not __restrict__:
// in place, every element is read by the lane that later overwrites it, and by no other.
// With kRope the normalised, affine-transformed q / k of a patch row are rotated (rope.cuh) before the one rounding.
template <int kVpl, bool kRope>
__device__ __forceinline__ void qk_norm_fwd_body(
    const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ bq,
    const __nv_bfloat16* __restrict__ wk, const __nv_bfloat16* __restrict__ bk, __nv_bfloat16* out, int64_t ld_out,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int H, int hd, int slots, int tokens_per_cta,
    float eps, const RopeArgs& rope) {
    constexpr int kTok = kVpl <= 2 ? 2 : 1;  // tokens whose loads are in flight together
    const int g = threadIdx.x / kQkLanes, lane = threadIdx.x % kQkLanes;
    const int j = blockIdx.x * kQkGroups + g;
    if (j >= slots) return;
    const unsigned mask = group_mask<kQkLanes>();
    const int nvec = hd / 8;
    const bool is_v = j >= 2 * H;
    const bool is_k = j >= H;
    uint4 gm[kVpl], bt[kVpl];
#pragma unroll
    for (int i = 0; i < kVpl; ++i) {
        const int idx = lane + i * kQkLanes;
        const bool ok = idx < nvec && !is_v;
        gm[i] = ok ? __ldg(reinterpret_cast<const uint4*>(is_k ? wk : wq) + idx) : make_uint4(0, 0, 0, 0);
        bt[i] = ok ? __ldg(reinterpret_cast<const uint4*>(is_k ? bk : bq) + idx) : make_uint4(0, 0, 0, 0);
    }
    const float inv_hd = 1.0f / static_cast<float>(hd);
    const int64_t t0 = static_cast<int64_t>(blockIdx.y) * tokens_per_cta;
    const int64_t t1 = min(static_cast<int64_t>(T), t0 + tokens_per_cta);

    auto row = [&](const uint4 (&v)[kVpl], int64_t t) {
        __nv_bfloat16* dst = out + t * ld_out + static_cast<int64_t>(j) * hd;
        if (is_v) {
#pragma unroll
            for (int i = 0; i < kVpl; ++i) {
                const int idx = lane + i * kQkLanes;
                if (idx < nvec) reinterpret_cast<uint4*>(dst)[idx] = v[i];
            }
            return;
        }
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < kVpl; ++i) {
            float f[8];
            qk_unpack8(v[i], f);  // vectors past the head are zero
#pragma unroll
            for (int q = 0; q < 8; ++q) s += f[q];
        }
        const float mean = group_sum<kQkLanes>(s, mask) * inv_hd;
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < kVpl; ++i) {
            if (lane + i * kQkLanes < nvec) {
                float f[8];
                qk_unpack8(v[i], f);
#pragma unroll
                for (int q = 0; q < 8; ++q) ss += (f[q] - mean) * (f[q] - mean);
            }
        }
        const float rstd = rsqrtf(group_sum<kQkLanes>(ss, mask) * inv_hd + eps);
        const int n = kRope ? rope_row(rope, static_cast<int>(t)) : -1;
#pragma unroll
        for (int i = 0; i < kVpl; ++i) {
            const int idx = lane + i * kQkLanes;
            if (idx < nvec) {
                float f[8], w[8], b[8];
                qk_unpack8(v[i], f);
                qk_unpack8(gm[i], w);
                qk_unpack8(bt[i], b);
#pragma unroll
                for (int q = 0; q < 8; ++q) f[q] = (f[q] - mean) * rstd * w[q] + b[q];
                if (kRope && n >= 0) rope_rotate<false>(f, rope, n, hd / 2, idx * 4);
                reinterpret_cast<uint4*>(dst)[idx] = qk_pack8(f);
            }
        }
        if (lane == 0) {
            mean_out[t * 2 * H + j] = mean;
            rstd_out[t * 2 * H + j] = rstd;
        }
    };

    for (int64_t t = t0; t < t1; t += kTok) {
        const int n = static_cast<int>(min(static_cast<int64_t>(kTok), t1 - t));  // group-uniform
        uint4 v[kTok][kVpl];
#pragma unroll
        for (int u = 0; u < kTok; ++u) {
            const uint4* src = reinterpret_cast<const uint4*>(qkv + (t + u) * ld + static_cast<int64_t>(j) * hd);
#pragma unroll
            for (int i = 0; i < kVpl; ++i) {
                const int idx = lane + i * kQkLanes;
                v[u][i] = (u < n && idx < nvec) ? src[idx] : make_uint4(0, 0, 0, 0);
            }
        }
#pragma unroll
        for (int u = 0; u < kTok; ++u)
            if (u < n) row(v[u], t + u);
    }
}

template <int kVpl>
__global__ void __launch_bounds__(kQkThreads) qk_norm_fwd_kernel(
    const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ bq,
    const __nv_bfloat16* __restrict__ wk, const __nv_bfloat16* __restrict__ bk, __nv_bfloat16* out, int64_t ld_out,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int H, int hd, int slots, int tokens_per_cta,
    float eps) {
    qk_norm_fwd_body<kVpl, false>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean_out, rstd_out, T, H, hd, slots,
                                  tokens_per_cta, eps, RopeArgs());
}
template <int kVpl>
__global__ void __launch_bounds__(kQkThreads) qk_norm_rope_fwd_kernel(
    const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ bq,
    const __nv_bfloat16* __restrict__ wk, const __nv_bfloat16* __restrict__ bk, __nv_bfloat16* out, int64_t ld_out,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, int T, int H, int hd, int slots, int tokens_per_cta,
    float eps, RopeArgs rope) {
    qk_norm_fwd_body<kVpl, true>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean_out, rstd_out, T, H, hd, slots,
                                 tokens_per_cta, eps, rope);
}

// In place on dqkv[:, 0:2D): the gradient of the normalised q / k becomes that of the un-normalised q / k (the standard
// LayerNorm backward on xhat = (x - mean) * rstd, x read from qkv).  dw / db: fp32 [hd] sums over all T * H rows of the
// side, reduced per CTA in shared memory and added with one atomic per column per CTA.  colsum[0, 2D): fp32 column sums
// of the stored bf16 dq / dk (the q / k part of the qkv bias gradient); every group of a CTA owns its own head slot, so
// each column gets one atomic per CTA.  All accumulators are added to: zero them first.
// With kRope the incoming dq / dk of a patch row are the gradients of the rotated values: R^T turns them, in fp32
// registers, into the gradients of the normalised ones before anything else reads them.
template <int kLanes, int kVpl, bool kRope>
__device__ __forceinline__ void qk_norm_bwd_body(
    __nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* __restrict__ qkv, int64_t ld,
    const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ wk, const float* __restrict__ mean,
    const float* __restrict__ rstd, float* __restrict__ dwq, float* __restrict__ dbq, float* __restrict__ dwk,
    float* __restrict__ dbk, float* __restrict__ colsum, int T, int H, int hd, int tokens_per_cta,
    const RopeArgs& rope) {
    constexpr int kGroups = kQkThreads / kLanes;
    __shared__ float red[4][kQkMaxHd];  // dw_q, db_q, dw_k, db_k of this CTA
    for (int i = threadIdx.x; i < 4 * kQkMaxHd; i += kQkThreads) (&red[0][0])[i] = 0.f;
    __syncthreads();
    const int g = threadIdx.x / kLanes, lane = threadIdx.x % kLanes;
    const int j = blockIdx.x * kGroups + g;
    const int nvec = hd / 8;
    if (j < 2 * H) {
        const unsigned mask = group_mask<kLanes>();
        const bool is_k = j >= H;
        uint4 gm[kVpl];
#pragma unroll
        for (int i = 0; i < kVpl; ++i) {
            const int idx = lane + i * kLanes;
            gm[i] = idx < nvec ? __ldg(reinterpret_cast<const uint4*>(is_k ? wk : wq) + idx) : make_uint4(0, 0, 0, 0);
        }
        float aw[kVpl][8], ab[kVpl][8], ac[kVpl][8];
#pragma unroll
        for (int i = 0; i < kVpl; ++i)
#pragma unroll
            for (int q = 0; q < 8; ++q) aw[i][q] = ab[i][q] = ac[i][q] = 0.f;
        const float inv_hd = 1.0f / static_cast<float>(hd);
        const int64_t t0 = static_cast<int64_t>(blockIdx.y) * tokens_per_cta;
        const int64_t t1 = min(static_cast<int64_t>(T), t0 + tokens_per_cta);

        auto row = [&](const uint4 (&xv)[kVpl], const uint4 (&dv)[kVpl], int64_t t) {
            const float m = __ldg(mean + t * 2 * H + j), r = __ldg(rstd + t * 2 * H + j);
            const int n = kRope ? rope_row(rope, static_cast<int>(t)) : -1;
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int i = 0; i < kVpl; ++i) {
                float x[8], dy[8], w[8];
                qk_unpack8(xv[i], x);
                qk_unpack8(dv[i], dy);  // zero past the head: those columns add nothing
                if (kRope && n >= 0 && lane + i * kLanes < nvec) rope_rotate<true>(dy, rope, n, hd / 2, (lane + i * kLanes) * 4);
                qk_unpack8(gm[i], w);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float xh = (x[q] - m) * r, gy = dy[q] * w[q];
                    s1 += gy;
                    s2 += gy * xh;
                    aw[i][q] += dy[q] * xh;
                    ab[i][q] += dy[q];
                }
            }
            s1 = group_sum<kLanes>(s1, mask) * inv_hd;
            s2 = group_sum<kLanes>(s2, mask) * inv_hd;
            __nv_bfloat16* dst = dqkv + t * ld_d + static_cast<int64_t>(j) * hd;
#pragma unroll
            for (int i = 0; i < kVpl; ++i) {
                const int idx = lane + i * kLanes;
                if (idx < nvec) {
                    float x[8], dy[8], w[8];
                    qk_unpack8(xv[i], x);
                    qk_unpack8(dv[i], dy);
                    if (kRope && n >= 0) rope_rotate<true>(dy, rope, n, hd / 2, idx * 4);
                    qk_unpack8(gm[i], w);
#pragma unroll
                    for (int q = 0; q < 8; ++q) dy[q] = r * (dy[q] * w[q] - s1 - (x[q] - m) * r * s2);
                    const uint4 o = qk_pack8(dy);
                    reinterpret_cast<uint4*>(dst)[idx] = o;
                    qk_unpack8(o, dy);  // the column sums are those of the rounded gradient the GEMMs consume
#pragma unroll
                    for (int q = 0; q < 8; ++q) ac[i][q] += dy[q];
                }
            }
        };

        for (int64_t t = t0; t < t1; ++t) {
            uint4 xv[kVpl], dv[kVpl];
            const uint4* xs = reinterpret_cast<const uint4*>(qkv + t * ld + static_cast<int64_t>(j) * hd);
            const uint4* ds = reinterpret_cast<const uint4*>(dqkv + t * ld_d + static_cast<int64_t>(j) * hd);
#pragma unroll
            for (int i = 0; i < kVpl; ++i) {
                const int idx = lane + i * kLanes;
                xv[i] = idx < nvec ? __ldg(xs + idx) : make_uint4(0, 0, 0, 0);
                dv[i] = idx < nvec ? ds[idx] : make_uint4(0, 0, 0, 0);
            }
            row(xv, dv, t);
        }
        float* rw = red[is_k ? 2 : 0];
        float* rb = red[is_k ? 3 : 1];
#pragma unroll
        for (int i = 0; i < kVpl; ++i) {
            const int idx = lane + i * kLanes;
            if (idx < nvec) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    atomicAdd(rw + idx * 8 + q, aw[i][q]);
                    atomicAdd(rb + idx * 8 + q, ab[i][q]);
                    atomicAdd(colsum + static_cast<int64_t>(j) * hd + idx * 8 + q, ac[i][q]);
                }
            }
        }
    }
    __syncthreads();
    const int jlo = blockIdx.x * kGroups, jhi = min(2 * H, jlo + kGroups);  // head slots of this CTA: [jlo, jhi)
    const bool has_q = jlo < H, has_k = jhi > H;
    for (int i = threadIdx.x; i < 4 * hd; i += kQkThreads) {
        const int side = i / hd, c = i % hd;
        if (side < 2 ? !has_q : !has_k) continue;
        float* dst = side == 0 ? dwq : side == 1 ? dbq : side == 2 ? dwk : dbk;
        atomicAdd(dst + c, red[side][c]);
    }
}

template <int kLanes, int kVpl>
__global__ void __launch_bounds__(kQkThreads) qk_norm_bwd_kernel(
    __nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* __restrict__ qkv, int64_t ld,
    const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ wk, const float* __restrict__ mean,
    const float* __restrict__ rstd, float* __restrict__ dwq, float* __restrict__ dbq, float* __restrict__ dwk,
    float* __restrict__ dbk, float* __restrict__ colsum, int T, int H, int hd, int tokens_per_cta) {
    qk_norm_bwd_body<kLanes, kVpl, false>(dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H, hd,
                                          tokens_per_cta, RopeArgs());
}
template <int kLanes, int kVpl>
__global__ void __launch_bounds__(kQkThreads, 2) qk_norm_rope_bwd_kernel(  // two CTAs per SM, as the plain kernel
    __nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* __restrict__ qkv, int64_t ld,
    const __nv_bfloat16* __restrict__ wq, const __nv_bfloat16* __restrict__ wk, const float* __restrict__ mean,
    const float* __restrict__ rstd, float* __restrict__ dwq, float* __restrict__ dbq, float* __restrict__ dwk,
    float* __restrict__ dbk, float* __restrict__ colsum, int T, int H, int hd, int tokens_per_cta, RopeArgs rope) {
    qk_norm_bwd_body<kLanes, kVpl, true>(dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H, hd,
                                         tokens_per_cta, rope);
}

inline void check_launch_qk(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

int sm_count_qk() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}

void check_qk_shapes(const char* what, int T, int H, int hd) {
    if (hd % 8 != 0 || hd < 8 || hd > kQkMaxHd)
        throw std::runtime_error(std::string(what) + ": head dim must be a multiple of 8 in [8, 256] (hd % 8 == 0 and "
                                 "8 <= hd <= 256), got " + std::to_string(hd));
    if (T < 0 || H < 1) throw std::runtime_error(std::string(what) + ": need T >= 0 and H >= 1");
}

void check_qk_matrix(const char* what, const char* name, const void* p, int64_t ld, int64_t width) {
    if ((reinterpret_cast<uintptr_t>(p) & 15) || ld % 8 != 0)
        throw std::runtime_error(std::string(what) + ": " + name + " must be 16-byte aligned with a leading dimension "
                                 "that is a multiple of 8 elements (16 bytes), got ld " + std::to_string(ld));
    if (ld < width)
        throw std::runtime_error(std::string(what) + ": " + name + " leading dimension " + std::to_string(ld) +
                                 " is narrower than 3 * H * hd = " + std::to_string(width));
}

// Token slabs: grid.y slabs of tokens_per tokens for grid.x head-slot chunks, about `ctas` CTAs in all.
void qk_grid(int T, int gx, int ctas, int& slabs, int& tokens_per) {
    slabs = std::max(1, std::min(std::min(T, 65535), ctas / gx));
    tokens_per = (T + slabs - 1) / slabs;
    slabs = (T + tokens_per - 1) / tokens_per;
}

}  // namespace

namespace {

// rope == nullptr: the plain kernels; otherwise the RoPE-fused instances, with B images of rope->tokens rows.
void qk_norm_fwd_launch(const char* what, const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq,
                        const __nv_bfloat16* bq, const __nv_bfloat16* wk, const __nv_bfloat16* bk, __nv_bfloat16* out,
                        int64_t ld_out, float* mean, float* rstd, int T, int H, int hd, float eps,
                        const RopeArgs* rope, cudaStream_t stream) {
    check_qk_shapes(what, T, H, hd);
    const int64_t width = 3 * static_cast<int64_t>(H) * hd;
    check_qk_matrix(what, "qkv", qkv, ld, width);
    check_qk_matrix(what, "out", out, ld_out, width);
    for (const void* p : {static_cast<const void*>(wq), static_cast<const void*>(bq), static_cast<const void*>(wk),
                          static_cast<const void*>(bk)})
        if (reinterpret_cast<uintptr_t>(p) & 15) throw std::runtime_error(std::string(what) + ": weights must be 16-byte aligned");
    const bool in_place = out == qkv;
    if (in_place && ld_out != ld) throw std::runtime_error(std::string(what) + ": in place needs ld_out == ld");
    if (T == 0) return;
    const int slots = (in_place ? 2 : 3) * H;
    const int gx = (slots + kQkGroups - 1) / kQkGroups;
    int slabs, tokens_per;
    qk_grid(T, gx, sm_count_qk() * 32, slabs, tokens_per);
    const dim3 grid(gx, slabs);
    if (rope) {
        switch ((hd / 8 + kQkLanes - 1) / kQkLanes) {
            case 1: qk_norm_rope_fwd_kernel<1><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps, *rope); break;
            case 2: qk_norm_rope_fwd_kernel<2><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps, *rope); break;
            case 3: qk_norm_rope_fwd_kernel<3><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps, *rope); break;
            default: qk_norm_rope_fwd_kernel<4><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps, *rope); break;
        }
    } else {
        switch ((hd / 8 + kQkLanes - 1) / kQkLanes) {
            case 1: qk_norm_fwd_kernel<1><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps); break;
            case 2: qk_norm_fwd_kernel<2><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps); break;
            case 3: qk_norm_fwd_kernel<3><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps); break;
            default: qk_norm_fwd_kernel<4><<<grid, kQkThreads, 0, stream>>>(qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, slots, tokens_per, eps); break;
        }
    }
    check_launch_qk(what);
}

void qk_norm_bwd_launch(const char* what, __nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* qkv, int64_t ld,
                        const __nv_bfloat16* wq, const __nv_bfloat16* wk, const float* mean, const float* rstd,
                        float* dwq, float* dbq, float* dwk, float* dbk, float* colsum, int T, int H, int hd,
                        const RopeArgs* rope, cudaStream_t stream) {
    check_qk_shapes(what, T, H, hd);
    const int64_t width = 3 * static_cast<int64_t>(H) * hd;
    check_qk_matrix(what, "dqkv", dqkv, ld_d, width);
    check_qk_matrix(what, "qkv", qkv, ld, width);
    if ((reinterpret_cast<uintptr_t>(wq) | reinterpret_cast<uintptr_t>(wk)) & 15)
        throw std::runtime_error(std::string(what) + ": weights must be 16-byte aligned");
    if (T == 0) return;
    // Three builds keep the three fp32 accumulators of each lane (dw, db, colsum) in at most 2 x 8 columns, so that two
    // CTAs fit an SM without spills: 8 lanes x 1 vector (hd <= 64), 8 x 2 (hd <= 128), 16 x 2 (hd <= 256).
    const int nvec = hd / 8;
    const int lanes = nvec > 16 ? 16 : 8;
    const int gx = (2 * H + kQkThreads / lanes - 1) / (kQkThreads / lanes);
    int slabs, tokens_per;
    qk_grid(T, gx, sm_count_qk() * 2, slabs, tokens_per);  // one resident wave: few dw / db atomics
    const dim3 grid(gx, slabs);
#define QK_BWD(L, V) qk_norm_bwd_kernel<L, V><<<grid, kQkThreads, 0, stream>>>(dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H, hd, tokens_per)
#define QK_ROPE_BWD(L, V) qk_norm_rope_bwd_kernel<L, V><<<grid, kQkThreads, 0, stream>>>(dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H, hd, tokens_per, *rope)
    if (rope) {
        if (nvec <= 8) QK_ROPE_BWD(8, 1);
        else if (nvec <= 16) QK_ROPE_BWD(8, 2);
        else QK_ROPE_BWD(16, 2);
    } else {
        if (nvec <= 8) QK_BWD(8, 1);
        else if (nvec <= 16) QK_BWD(8, 2);
        else QK_BWD(16, 2);
    }
#undef QK_ROPE_BWD
#undef QK_BWD
    check_launch_qk(what);
}

}  // namespace

void qk_norm_fwd(const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq, const __nv_bfloat16* bq,
                 const __nv_bfloat16* wk, const __nv_bfloat16* bk, __nv_bfloat16* out, int64_t ld_out, float* mean,
                 float* rstd, int T, int H, int hd, float eps, cudaStream_t stream) {
    qk_norm_fwd_launch("qk_norm_fwd", qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, eps, nullptr, stream);
}

void qk_norm_bwd(__nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq,
                 const __nv_bfloat16* wk, const float* mean, const float* rstd, float* dwq, float* dbq, float* dwk,
                 float* dbk, float* colsum, int T, int H, int hd, cudaStream_t stream) {
    qk_norm_bwd_launch("qk_norm_bwd", dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H, hd,
                       nullptr, stream);
}

void qk_norm_rope_fwd(const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq, const __nv_bfloat16* bq,
                      const __nv_bfloat16* wk, const __nv_bfloat16* bk, __nv_bfloat16* out, int64_t ld_out,
                      float* mean, float* rstd, const RopeArgs& rope, int B, int H, int hd, float eps,
                      cudaStream_t stream) {
    check_rope_args("qk_norm_rope_fwd", rope, B, H, hd);  // also: B * tokens fits 32 bits
    const int T = B * rope.tokens;
    qk_norm_fwd_launch("qk_norm_rope_fwd", qkv, ld, wq, bq, wk, bk, out, ld_out, mean, rstd, T, H, hd, eps, &rope,
                       stream);
}

void qk_norm_rope_bwd(__nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* qkv, int64_t ld,
                      const __nv_bfloat16* wq, const __nv_bfloat16* wk, const float* mean, const float* rstd,
                      float* dwq, float* dbq, float* dwk, float* dbk, float* colsum, const RopeArgs& rope, int B,
                      int H, int hd, cudaStream_t stream) {
    check_rope_args("qk_norm_rope_bwd", rope, B, H, hd);  // also: B * tokens fits 32 bits
    const int T = B * rope.tokens;
    qk_norm_bwd_launch("qk_norm_rope_bwd", dqkv, ld_d, qkv, ld, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, colsum, T, H,
                       hd, &rope, stream);
}

}  // namespace b200
