// LayerNorm backward for wide rows (D >= 2048) as a bulk-copy pipeline.
//
// The register-resident kernel in elementwise.cu pays, per row, a shared-memory read-modify-write of 3 x D column
// accumulators, two block barriers and a half-empty third chunk (D = 5120 over 256 threads): many instructions per
// byte moved.  (Neither kernel has been timed on H100.)  This version:
//   * one producer thread streams whole rows (x, dy, residual gradient: one cp.async.bulk each, 10 KB at D = 5120)
//     into a shared-memory ring of kStages rows, completion on mbarriers -- 90+ KB in flight per SM with zero
//     register cost, so a single CTA per SM saturates HBM;
//   * D / 16 consumer threads own 16 columns each for the whole kernel: dgamma / dbeta / dx column sums stay in
//     REGISTERS (48 accumulators), gamma is loaded once;
//   * one named barrier per row (double-buffered partial sums) for the two row reductions
//         s1 = sum_j dy_j g_j,   s2 = sum_j dy_j g_j (x_j - mean)
//     (s2 on centred x) and dx folded into two FMAs per element:  dx = dres + (rstd g) dy - k1 x + k0 with per-row
//     constants k1, k0, so the second pass over the row (re-read from shared memory, not from HBM) is short.
// dx = [dres +] rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)), dgamma += sum_rows dy*xhat, dbeta += sum_rows dy,
// dxsum += sum_rows dx (the bias gradient of the Linear that produced x's residual branch).
// Reference op: autograd through nn.LayerNorm in timm Block / the final norm (run_vit_training.py:134-141,151).
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

#include "elementwise.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kVPT = 2;     // 16-byte vectors (8 bf16 columns) per consumer thread
constexpr int kStages = 4;  // rows in flight per CTA

__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    f[0] = bf16_lo(v.x), f[1] = bf16_hi(v.x), f[2] = bf16_lo(v.y), f[3] = bf16_hi(v.y);
    f[4] = bf16_lo(v.z), f[5] = bf16_hi(v.z), f[6] = bf16_lo(v.w), f[7] = bf16_hi(v.w);
}

template <bool kRes, bool kDxSum, int kMaxThreads>
__global__ void __launch_bounds__(kMaxThreads, 1)
    ln_bwd_stream_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                         const __nv_bfloat16* __restrict__ gamma, const float* __restrict__ mean_in,
                         const float* __restrict__ rstd_in, const __nv_bfloat16* __restrict__ dres,
                         __nv_bfloat16* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                         float* __restrict__ dxsum, int rows, int D) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int row_bytes = D * 2;
    constexpr int kTensors = kRes ? 3 : 2;
    const int stage_bytes = kTensors * row_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * stage_bytes);
    uint64_t* empty = full + kStages;
    float* red = reinterpret_cast<float*>(empty + kStages);  // [2][consumer warps][2]

    const int ncons = static_cast<int>(blockDim.x) - 32;  // consumer threads = D / (8 * kVPT)
    const int ncw = ncons / 32;
    const int tid = threadIdx.x;
    const int n_my = (rows - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);

    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], ncw);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (tid < 32) {
        // ===================================== producer =====================================
        if (tid == 0) {
            for (int it = 0; it < n_my; ++it) {
                const int st = it % kStages;
                if (it >= kStages) mbar_wait(&empty[st], ((it / kStages) - 1) & 1);
                const int64_t row = static_cast<int64_t>(blockIdx.x) + static_cast<int64_t>(it) * gridDim.x;
                uint8_t* dst = smem + st * stage_bytes;
                mbar_arrive_expect_tx(&full[st], stage_bytes);
                bulk_load(dst, x + row * D, row_bytes, &full[st]);
                bulk_load(dst + row_bytes, dy + row * D, row_bytes, &full[st]);
                if constexpr (kRes) bulk_load(dst + 2 * row_bytes, dres + row * D, row_bytes, &full[st]);
            }
        }
        return;
    }

    // ===================================== consumers =====================================
    const int ct = tid - 32;          // consumer thread index
    const int cw = ct / 32;           // consumer warp
    const int lane = ct % 32;
    const float inv_d = 1.0f / static_cast<float>(D);
    float gam[kVPT][8], dg[kVPT][8], db[kVPT][8], dxs[kVPT][8];
#pragma unroll
    for (int v = 0; v < kVPT; ++v) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(gamma) + ct + v * ncons), gam[v]);
#pragma unroll
        for (int q = 0; q < 8; ++q) dg[v][q] = 0.f, db[v][q] = 0.f, dxs[v][q] = 0.f;
    }
    for (int it = 0; it < n_my; ++it) {
        const int st = it % kStages;
        const int64_t row = static_cast<int64_t>(blockIdx.x) + static_cast<int64_t>(it) * gridDim.x;
        const float mean = __ldg(mean_in + row), rstd = __ldg(rstd_in + row);
        mbar_wait(&full[st], (it / kStages) & 1);
        const uint4* sx = reinterpret_cast<const uint4*>(smem + st * stage_bytes);
        const uint4* sdy = reinterpret_cast<const uint4*>(smem + st * stage_bytes + row_bytes);
        const uint4* sres = reinterpret_cast<const uint4*>(smem + st * stage_bytes + 2 * row_bytes);
        // ---- pass A: row sums + column accumulators that do not need them ----
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int v = 0; v < kVPT; ++v) {
            float xf[8], df[8];
            unpack8(sx[ct + v * ncons], xf);
            unpack8(sdy[ct + v * ncons], df);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float t = df[q] * gam[v][q];
                const float xm = xf[q] - mean;  // centred first: no cancellation when |mean| >> std
                s1 += t;
                s2 = fmaf(t, xm, s2);
                dg[v][q] = fmaf(df[q] * rstd, xm, dg[v][q]);
                db[v][q] += df[q];
            }
        }
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        float* rbuf = red + (it & 1) * (2 * ncw);
        if (lane == 0) {
            rbuf[cw * 2] = s1;
            rbuf[cw * 2 + 1] = s2;
        }
        named_bar_sync(1, ncons);
        float t1 = 0.f, t2 = 0.f;
        for (int w = 0; w < ncw; ++w) {
            t1 += rbuf[w * 2];
            t2 += rbuf[w * 2 + 1];
        }
        // t1 = sum_j g dy, t2 = sum_j g dy (x - mean):  mean_j(g dy) = t1/D ; mean_j(g dy xhat) = rstd t2/D
        // dx = dres + rstd*(g dy) - rstd*m1 - rstd*xhat*m2 = dres + rstd*(g dy) - k1*x + k0
        const float m1 = t1 * inv_d;
        const float m2 = rstd * t2 * inv_d;
        const float k1 = rstd * rstd * m2;
        const float k0 = k1 * mean - rstd * m1;
        // ---- pass B: dx (the row is still in shared memory) ----
        uint4* dxr = reinterpret_cast<uint4*>(dx + row * D);
#pragma unroll
        for (int v = 0; v < kVPT; ++v) {
            float xf[8], df[8], rf[8], o[8];
            unpack8(sx[ct + v * ncons], xf);
            unpack8(sdy[ct + v * ncons], df);
            if constexpr (kRes) {
                unpack8(sres[ct + v * ncons], rf);
            } else {
#pragma unroll
                for (int q = 0; q < 8; ++q) rf[q] = 0.f;
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                float r = fmaf(rstd * gam[v][q], df[q], rf[q] + k0);
                r = fmaf(-k1, xf[q], r);
                o[q] = r;
            }
            uint4 pk;
            pk.x = pack_bf16x2(o[0], o[1]), pk.y = pack_bf16x2(o[2], o[3]);
            pk.z = pack_bf16x2(o[4], o[5]), pk.w = pack_bf16x2(o[6], o[7]);
            dxr[ct + v * ncons] = pk;
            if constexpr (kDxSum) {
                unpack8(pk, o);  // sum what was stored (bf16-rounded), as ln_bwd_kernel and the GEMM colsum do
#pragma unroll
                for (int q = 0; q < 8; ++q) dxs[v][q] += o[q];
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);  // this warp no longer reads the stage
    }
    // one global atomic per column per CTA (one arrival per SM per address)
#pragma unroll
    for (int v = 0; v < kVPT; ++v) {
        const int c0 = (ct + v * ncons) * 8;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            atomicAdd(dgamma + c0 + q, dg[v][q]);
            atomicAdd(dbeta + c0 + q, db[v][q]);
            if constexpr (kDxSum) atomicAdd(dxsum + c0 + q, dxs[v][q]);
        }
    }
}

int sm_count_ln() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}

template <bool kRes, bool kDxSum, int kMaxThreads>
void launch_stream_t(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                   const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                   float* dxsum, int rows, int D, cudaStream_t stream) {
    const int ncons = D / (8 * kVPT);
    const size_t smem = static_cast<size_t>(kStages) * (kRes ? 3 : 2) * D * 2 + 2 * kStages * 8 + 2 * 2 * (ncons / 32) * 4 + 64;
    auto kern = ln_bwd_stream_kernel<kRes, kDxSum, kMaxThreads>;
    static size_t attr = 0;
    if (smem > attr) {
        cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
        if (err != cudaSuccess) throw std::runtime_error(std::string("ln_bwd_stream smem attr: ") + cudaGetErrorString(err));
        attr = smem;
    }
    const int grid = std::min(rows, sm_count_ln());
    kern<<<grid, 32 + ncons, smem, stream>>>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string("ln_bwd_stream launch: ") + cudaGetErrorString(err));
}

template <bool kRes, bool kDxSum>
void launch_stream(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                   const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                   float* dxsum, int rows, int D, cudaStream_t stream) {
    // D <= 5632 (ViT-10B: 5120 -> 352 threads) gets the 384-thread build with a 168-register budget (no spills)
    if (32 + D / (8 * kVPT) <= 384)
        launch_stream_t<kRes, kDxSum, 384>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
    else
        launch_stream_t<kRes, kDxSum, 672>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
}

}  // namespace

bool layernorm_bwd_stream_supported(int D) {
    // whole consumer warps, at most 640 consumer threads, 4 stages of up to 3 rows within 227 KB of shared memory
    return D % (8 * kVPT * 32) == 0 && D / (8 * kVPT) <= 640 && D >= 2048 &&
           static_cast<size_t>(kStages) * 3 * D * 2 + 1024 <= 232448;
}

void layernorm_bwd_stream(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                          const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                          float* dxsum, int rows, int D, cudaStream_t stream) {
    if (!layernorm_bwd_stream_supported(D)) throw std::runtime_error("layernorm_bwd_stream: unsupported width");
    if (dres != nullptr) {
        if (dxsum != nullptr) launch_stream<true, true>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
        else launch_stream<true, false>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
    } else {
        if (dxsum != nullptr) launch_stream<false, true>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
        else launch_stream<false, false>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, rows, D, stream);
    }
}

}  // namespace b200
