// Patch dropout (timm PatchDropout(prob=R, num_prefix_tokens=P, ordered=True), Liu et al. 2022): in training every image
// keeps K = max(1, int(N * (1 - R))) of its N patch tokens, so every block runs on T' = P + K tokens.
//
// patch_drop_select: one CTA per image.  It draws r[n] for its N patches (word n % 4 of philox4x32_10(n / 4, g, key),
//   image g = offset + b), bitonic-sorts the 64-bit keys (r << 32) | n in shared memory (the order is total: ties break
//   on n), flags the first K, and a block-wide prefix scan over the flags writes keep in ascending patch order and inv.
// im2col_gather_kernel: the patch im2col of the kept patches only (the pixel fetch and batch mixing are im2col_kernel's,
//   im2col_pixel.cuh), so only they go through the patch GEMM.
// pos_gather_kernel: the position rows of the kept patches, a 16-byte vector copy; the patch GEMM adds them as its
//   residual in fp32 together with the bias, as on the full-sequence path.
// patch_drop_bwd_kernel: one thread per (token j of the full sequence, 8 columns), modelled on tokens_bwd_kernel; it
//   walks b = 0 .. B-1 in order and reads each kept row of dx0 exactly once.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "dropout.cuh"
#include "im2col_pixel.cuh"
#include "patch_drop.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kSelThreads = 1024;
constexpr int kPdThreads = 256;
constexpr int kPdUnroll = 4;  // 16-byte vectors per thread in flight

__global__ void __launch_bounds__(kSelThreads) patch_drop_select_kernel(int* __restrict__ keep, int* __restrict__ inv,
                                                                        int N, int K, int npow2, uint32_t g0,
                                                                        uint32_t key_lo, uint32_t key_hi) {
    extern __shared__ uint64_t sel_keys[];                            // [npow2]
    uint8_t* flag = reinterpret_cast<uint8_t*>(sel_keys + npow2);     // [N]
    __shared__ int warp_tot[kSelThreads / 32];
    const int tid = threadIdx.x, b = blockIdx.x;
    const uint32_t g = g0 + static_cast<uint32_t>(b);
    for (int q = tid; q < npow2 / 4; q += kSelThreads) {
        uint32_t r[4];
        philox4x32_10(static_cast<uint32_t>(q), g, key_lo, key_hi, r);
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const int n = 4 * q + w;
            sel_keys[n] = n < N ? (static_cast<uint64_t>(r[w]) << 32) | static_cast<uint32_t>(n) : ~0ull;
        }
    }
    for (int n = tid; n < N; n += kSelThreads) flag[n] = 0;
    __syncthreads();
    for (int k = 2; k <= npow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < npow2; i += kSelThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t a = sel_keys[i], c = sel_keys[ixj];
                    if ((a > c) == ((i & k) == 0)) {
                        sel_keys[i] = c;
                        sel_keys[ixj] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < K; i += kSelThreads) flag[static_cast<uint32_t>(sel_keys[i])] = 1;
    __syncthreads();
    // thread t owns the patches [t * per, (t + 1) * per): local count, block-wide exclusive scan, then the writes
    const int per = (N + kSelThreads - 1) / kSelThreads;
    const int n0 = min(N, tid * per), n1 = min(N, n0 + per);
    int cnt = 0;
    for (int n = n0; n < n1; ++n) cnt += flag[n];
    const int lane = tid & 31, wid = tid >> 5;
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int t = warp_tot[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += v;
        }
        warp_tot[lane] = t;  // inclusive totals of warps 0 .. lane
    }
    __syncthreads();
    int pos = incl - cnt + (wid > 0 ? warp_tot[wid - 1] : 0);
    int* keep_b = keep + static_cast<int64_t>(b) * K;
    int* inv_b = inv + static_cast<int64_t>(b) * N;
    for (int n = n0; n < n1; ++n) {
        if (flag[n]) {
            keep_b[pos] = n;
            inv_b[n] = pos++;
        } else {
            inv_b[n] = -1;
        }
    }
}

template <typename T, int MIX>
__global__ void im2col_gather_kernel(const T* __restrict__ img, const int* __restrict__ keep,
                                     __nv_bfloat16* __restrict__ cols, int B, int S, int P, int Kpad, int K,
                                     Im2colMix mix) {
    // 32-bit index math throughout (the host checks B * K * Kpad < 2^31)
    const int G = S / P;
    const int total = B * K * Kpad;
    const int K3 = 3 * P * P;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int row = i / Kpad, k = i - row * Kpad;
        float v = 0.f;
        if (k < K3) {
            const int patch = row / K * G * G + __ldg(keep + row);
            v = im2col_pixel<T, MIX>(img, B, S, P, G, patch, k, mix);
        }
        cols[i] = __float2bfloat16(v);
    }
}

__global__ void __launch_bounds__(kPdThreads) pos_gather_kernel(const uint4* __restrict__ pos,
                                                               const int* __restrict__ keep, uint4* __restrict__ out,
                                                               int rows, int D8) {
    const int idx = blockIdx.x * kPdThreads + threadIdx.x;
    if (idx >= rows * D8) return;
    const int r = idx / D8, c = idx - r * D8;
    out[idx] = __ldg(pos + static_cast<int64_t>(__ldg(keep + r)) * D8 + c);
}

__global__ void __launch_bounds__(kPdThreads) patch_drop_bwd_kernel(
    const uint4* __restrict__ dx0, const int* __restrict__ inv, uint4* __restrict__ dpatch, float4* __restrict__ dtok,
    int B, int N, int K, int P, int D8) {
    const int idx = blockIdx.x * kPdThreads + threadIdx.x;
    if (idx >= (P + N) * D8) return;
    const int j = idx / D8, c = idx - j * D8;
    const int T = P + K;
    const int n = j - P;  // the patch of row j (j >= P)
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int b0 = 0; b0 < B; b0 += kPdUnroll) {
        int row[kPdUnroll];  // row of image b0 + u within its kept sequence, -1 when absent
        uint4 v[kPdUnroll];
#pragma unroll
        for (int u = 0; u < kPdUnroll; ++u) {
            const int b = b0 + u;
            row[u] = b >= B ? -1 : (j < P ? j : __ldg(inv + static_cast<int64_t>(b) * N + n));
            if (row[u] >= 0 && j >= P) row[u] += P;
        }
#pragma unroll
        for (int u = 0; u < kPdUnroll; ++u)
            v[u] = row[u] >= 0 ? __ldg(dx0 + (static_cast<int64_t>(b0 + u) * T + row[u]) * D8 + c)
                               : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int u = 0; u < kPdUnroll; ++u) {
            if (row[u] < 0) continue;
            const uint32_t* vs = &v[u].x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                acc[2 * k] += bf16_lo(vs[k]);
                acc[2 * k + 1] += bf16_hi(vs[k]);
            }
            if (dpatch != nullptr && j >= P)
                dpatch[(static_cast<int64_t>(b0 + u) * K + row[u] - P) * D8 + c] = v[u];
        }
    }
    dtok[2 * static_cast<int64_t>(idx)] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dtok[2 * static_cast<int64_t>(idx) + 1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

void check_keep(const char* what, int64_t B, int64_t N, int64_t K) {
    const std::string w(what);
    if (B < 1) throw std::runtime_error(w + ": need B >= 1 images, got B " + std::to_string(B));
    if (N < 1 || N > kPatchDropMaxN)
        throw std::runtime_error(w + ": need 1 <= N <= " + std::to_string(kPatchDropMaxN) + " patches, got N " +
                                 std::to_string(N));
    if (K < 1 || K > N)
        throw std::runtime_error(w + ": need 1 <= K <= N kept patches, got K " + std::to_string(K) + ", N " +
                                 std::to_string(N));
    if (B * N > 0x7FFFFFFF) throw std::runtime_error(w + ": B * N too large for 32-bit row arithmetic");
}

void check_vec(const char* what, int64_t rows, int64_t D) {
    const std::string w(what);
    if (D < 8 || D % 8 != 0)
        throw std::runtime_error(w + ": need D % 8 == 0 (16-byte vectors), got D " + std::to_string(D));
    if (rows * (D / 8) > 0x7FFFFFFF) throw std::runtime_error(w + ": buffer too large for 32-bit row arithmetic");
}

void check_aligned_pd(const char* what, const char* name, const void* p) {
    if (reinterpret_cast<uintptr_t>(p) & 15)
        throw std::runtime_error(std::string(what) + ": " + name + " must be 16-byte aligned");
}

inline void check_launch_pd(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

template <typename T>
void im2col_gather_launch(const T* img, const int* keep, __nv_bfloat16* cols, int B, int S, int P, int Kpad, int K,
                          const Im2colMix& mix, cudaStream_t stream) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int total = B * K * Kpad;
    const int grid = std::min((total + 255) / 256, sms * 8);
    if (mix.mode == 0)
        im2col_gather_kernel<T, 0><<<grid, 256, 0, stream>>>(img, keep, cols, B, S, P, Kpad, K, mix);
    else if (mix.mode == 1)
        im2col_gather_kernel<T, 1><<<grid, 256, 0, stream>>>(img, keep, cols, B, S, P, Kpad, K, mix);
    else
        im2col_gather_kernel<T, 2><<<grid, 256, 0, stream>>>(img, keep, cols, B, S, P, Kpad, K, mix);
}

}  // namespace

void patch_drop_select(int* keep, int* inv, int64_t B, int64_t N, int64_t K, int64_t offset, uint64_t key,
                       cudaStream_t stream) {
    check_keep("patch_drop_select", B, N, K);
    if (offset < 0 || offset + B > (int64_t(1) << 32))
        throw std::runtime_error("patch_drop_select: need 0 <= offset and offset + B <= 2^32 (32-bit image counter)");
    int npow2 = 4;
    while (npow2 < N) npow2 <<= 1;
    // 36 KB at N = 4096, under the 48 KB a launch may take without an opt-in (with the 128-byte static scan buffer)
    const size_t smem = static_cast<size_t>(npow2) * sizeof(uint64_t) + static_cast<size_t>(N);
    patch_drop_select_kernel<<<static_cast<unsigned>(B), kSelThreads, smem, stream>>>(
        keep, inv, static_cast<int>(N), static_cast<int>(K), npow2, static_cast<uint32_t>(offset),
        static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32));
    check_launch_pd("patch_drop_select");
}

void im2col_gather(const void* img, bool img_is_bf16, const int* keep, __nv_bfloat16* cols, int B, int S, int P,
                   int Kpad, int K, cudaStream_t stream, const Im2colMix& mix) {
    if (P < 1 || S % P != 0) throw std::runtime_error("im2col_gather: the image size must be a multiple of the patch");
    check_keep("im2col_gather", B, static_cast<int64_t>(S / P) * (S / P), K);
    if (Kpad < 3 * P * P) throw std::runtime_error("im2col_gather: Kpad must be >= 3 P^2");
    if (static_cast<int64_t>(B) * K * Kpad > 0x7FFFFFFF)
        throw std::runtime_error("im2col_gather: B * K * Kpad too large for 32-bit index arithmetic");
    if (mix.mode < 0 || mix.mode > 2) throw std::runtime_error("im2col_gather: mix mode must be 0, 1 or 2");
    if (mix.mode != 0 && B % 2 != 0) throw std::runtime_error("im2col_gather: batch mixing needs an even batch");
    if (mix.mode == 2 && !(0 <= mix.yl && mix.yl <= mix.yh && mix.yh <= S && 0 <= mix.xl && mix.xl <= mix.xh &&
                           mix.xh <= S))
        throw std::runtime_error("im2col_gather: the CutMix box must lie inside the image");
    if (img_is_bf16)
        im2col_gather_launch(static_cast<const __nv_bfloat16*>(img), keep, cols, B, S, P, Kpad, K, mix, stream);
    else
        im2col_gather_launch(static_cast<const float*>(img), keep, cols, B, S, P, Kpad, K, mix, stream);
    check_launch_pd("im2col_gather");
}

void pos_gather(const __nv_bfloat16* pos, const int* keep, __nv_bfloat16* out, int64_t rows, int64_t D,
                cudaStream_t stream) {
    if (rows < 1) throw std::runtime_error("pos_gather: need at least one row");
    check_vec("pos_gather", rows, D);
    check_aligned_pd("pos_gather", "pos", pos);
    check_aligned_pd("pos_gather", "out", out);
    const int D8 = static_cast<int>(D / 8);
    const unsigned grid = static_cast<unsigned>((rows * D8 + kPdThreads - 1) / kPdThreads);
    pos_gather_kernel<<<grid, kPdThreads, 0, stream>>>(reinterpret_cast<const uint4*>(pos), keep,
                                                       reinterpret_cast<uint4*>(out), static_cast<int>(rows), D8);
    check_launch_pd("pos_gather");
}

void patch_drop_bwd(const __nv_bfloat16* dx0, const int* inv, __nv_bfloat16* dpatch, float* dtok, int64_t B,
                    int64_t N, int64_t K, int64_t P, int64_t D, cudaStream_t stream) {
    check_keep("patch_drop_bwd", B, N, K);
    if (P < 0) throw std::runtime_error("patch_drop_bwd: need P >= 0 prefix tokens, got P " + std::to_string(P));
    check_vec("patch_drop_bwd", B * (P + K) > P + N ? B * (P + K) : P + N, D);
    check_aligned_pd("patch_drop_bwd", "dx0", dx0);
    if (dpatch) check_aligned_pd("patch_drop_bwd", "dpatch", dpatch);
    check_aligned_pd("patch_drop_bwd", "dtok", dtok);
    const int D8 = static_cast<int>(D / 8);
    const unsigned grid = static_cast<unsigned>(((P + N) * D8 + kPdThreads - 1) / kPdThreads);
    patch_drop_bwd_kernel<<<grid, kPdThreads, 0, stream>>>(
        reinterpret_cast<const uint4*>(dx0), inv, reinterpret_cast<uint4*>(dpatch), reinterpret_cast<float4*>(dtok),
        static_cast<int>(B), static_cast<int>(N), static_cast<int>(K), static_cast<int>(P), D8);
    check_launch_pd("patch_drop_bwd");
}

}  // namespace b200
