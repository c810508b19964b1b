// Prefix tokens (timm VisionTransformer(class_token=True, reg_tokens=R)): every image's token sequence is
// [cls, reg_0 .. reg_{R-1}, patch_0 .. patch_{N-1}], T = N + P rows with P = 1 + R.  The patch GEMM keeps producing the
// patch rows y [B * N, D] with the bias and the patch rows of pos_embed added in its epilogue; these two memory-bound
// passes move them into / out of the [B * T, D] token buffer and handle the P prefix rows.
//
// tokens_fwd: one thread per 16-byte vector of x0.  A CTA owns a run of whole rows, so the row / column split is 32-bit
//   arithmetic; the prefix rows are prefix[j] (+ pos[j]) summed in fp32 and rounded once to bf16.
// tokens_bwd: one thread per (token j, 8 columns).  It walks the batch in order, b = 0 .. B-1, summing dx0[b * T + j]
//   in fp32 registers and copying patch rows to dpatch on the way: dtok needs no atomics and has the same bits in
//   every run.  At the ViT-10B shape (T = 257, D = 5120) that is 164 K threads with 4 loads each in flight.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <stdexcept>
#include <string>

#include "prefix_tokens.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kTokThreads = 256;
constexpr int kTokUnroll = 4;             // 16-byte vectors per thread in flight
constexpr int kFwdVecsPerCta = 2048;      // forward: about this many vectors (whole rows) per CTA

__global__ void __launch_bounds__(kTokThreads) tokens_fwd_kernel(
    const uint4* __restrict__ y, const uint4* __restrict__ cls, const uint4* __restrict__ reg,
    const uint4* __restrict__ pos, uint4* __restrict__ x0, int rows, int rows_per_cta, int T, int N, int P, int D8) {
    const int r0 = blockIdx.x * rows_per_cta;
    const int nrows = min(rows_per_cta, rows - r0);
    const int nvec = nrows * D8;
    for (int l0 = threadIdx.x; l0 < nvec; l0 += kTokThreads * kTokUnroll) {
        uint4 v[kTokUnroll];
#pragma unroll
        for (int u = 0; u < kTokUnroll; ++u) {
            const int l = l0 + u * kTokThreads;
            if (l >= nvec) break;
            const int r = r0 + l / D8, c = l % D8;
            const int b = r / T, j = r - b * T;
            if (j >= P) {
                v[u] = __ldg(y + ((int64_t)b * N + (j - P)) * D8 + c);
            } else {
                const uint4 t = __ldg((j == 0 ? cls : reg + (int64_t)(j - 1) * D8) + c);
                if (pos == nullptr) {
                    v[u] = t;
                } else {
                    const uint4 q = __ldg(pos + (int64_t)j * D8 + c);
                    const uint32_t* ts = &t.x;
                    const uint32_t* qs = &q.x;
                    uint32_t* vs = &v[u].x;
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        vs[k] = pack_bf16x2(bf16_lo(ts[k]) + bf16_lo(qs[k]), bf16_hi(ts[k]) + bf16_hi(qs[k]));
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kTokUnroll; ++u) {
            const int l = l0 + u * kTokThreads;
            if (l >= nvec) break;
            x0[(int64_t)r0 * D8 + l] = v[u];
        }
    }
}

__global__ void __launch_bounds__(kTokThreads) tokens_bwd_kernel(
    const uint4* __restrict__ dx0, uint4* __restrict__ dpatch, float4* __restrict__ dtok, int B, int T, int N, int P,
    int D8) {
    const int idx = blockIdx.x * kTokThreads + threadIdx.x;
    if (idx >= T * D8) return;
    const int j = idx / D8, c = idx - j * D8;
    const bool patch = j >= P;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    const int64_t stride = (int64_t)T * D8;  // one image
    const uint4* src = dx0 + (int64_t)j * D8 + c;
    uint4* dst = patch ? dpatch + (int64_t)(j - P) * D8 + c : nullptr;
    for (int b0 = 0; b0 < B; b0 += kTokUnroll) {
        uint4 v[kTokUnroll];
#pragma unroll
        for (int u = 0; u < kTokUnroll; ++u)
            v[u] = b0 + u < B ? __ldg(src + (b0 + u) * stride) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int u = 0; u < kTokUnroll; ++u) {
            if (b0 + u >= B) break;
            const uint32_t* vs = &v[u].x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                acc[2 * k] += bf16_lo(vs[k]);
                acc[2 * k + 1] += bf16_hi(vs[k]);
            }
            if (patch) dst[(int64_t)(b0 + u) * N * D8] = v[u];
        }
    }
    dtok[2 * (int64_t)idx] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dtok[2 * (int64_t)idx + 1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

void check_tok(const char* what, int64_t B, int64_t N, int64_t P, int64_t D) {
    const std::string w(what);
    if (P < 1) throw std::runtime_error(w + ": need P >= 1 prefix tokens, got P " + std::to_string(P));
    if (B < 1 || N < 1) throw std::runtime_error(w + ": need B >= 1 images and N >= 1 patches, got B " +
                                                 std::to_string(B) + ", N " + std::to_string(N));
    if (D < 8 || D % 8 != 0) throw std::runtime_error(w + ": need D % 8 == 0 (16-byte vectors), got D " +
                                                      std::to_string(D));
    if (B * (N + P) > 0x7FFFFFFF || (N + P) * (D / 8) > 0x7FFFFFFF || B * (N + P) * (D / 8) > (int64_t(1) << 40))
        throw std::runtime_error(w + ": token buffer too large for 32-bit row arithmetic");
}

void check_aligned(const char* what, const char* name, const void* p) {
    if (reinterpret_cast<uintptr_t>(p) & 15)
        throw std::runtime_error(std::string(what) + ": " + name + " must be 16-byte aligned");
}

inline void check_launch_tok(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

}  // namespace

void tokens_fwd(const __nv_bfloat16* y, const __nv_bfloat16* cls, const __nv_bfloat16* reg, const __nv_bfloat16* pos,
                __nv_bfloat16* x0, int64_t B, int64_t N, int64_t P, int64_t D, cudaStream_t stream) {
    check_tok("tokens_fwd", B, N, P, D);
    if (P > 1 && reg == nullptr) throw std::runtime_error("tokens_fwd: P > 1 needs the register tokens");
    check_aligned("tokens_fwd", "y", y);
    check_aligned("tokens_fwd", "cls", cls);
    if (reg) check_aligned("tokens_fwd", "reg", reg);
    if (pos) check_aligned("tokens_fwd", "pos", pos);
    check_aligned("tokens_fwd", "x0", x0);
    const int D8 = static_cast<int>(D / 8), T = static_cast<int>(N + P);
    const int rows = static_cast<int>(B * T);
    const int rows_per_cta = D8 >= kFwdVecsPerCta ? 1 : kFwdVecsPerCta / D8;
    const unsigned grid = static_cast<unsigned>((rows + rows_per_cta - 1) / rows_per_cta);
    tokens_fwd_kernel<<<grid, kTokThreads, 0, stream>>>(
        reinterpret_cast<const uint4*>(y), reinterpret_cast<const uint4*>(cls), reinterpret_cast<const uint4*>(reg),
        reinterpret_cast<const uint4*>(pos), reinterpret_cast<uint4*>(x0), rows, rows_per_cta, T,
        static_cast<int>(N), static_cast<int>(P), D8);
    check_launch_tok("tokens_fwd");
}

void tokens_bwd(const __nv_bfloat16* dx0, __nv_bfloat16* dpatch, float* dtok, int64_t B, int64_t N, int64_t P,
                int64_t D, cudaStream_t stream) {
    check_tok("tokens_bwd", B, N, P, D);
    check_aligned("tokens_bwd", "dx0", dx0);
    check_aligned("tokens_bwd", "dpatch", dpatch);
    check_aligned("tokens_bwd", "dtok", dtok);
    const int D8 = static_cast<int>(D / 8), T = static_cast<int>(N + P);
    const unsigned grid = static_cast<unsigned>((static_cast<int64_t>(T) * D8 + kTokThreads - 1) / kTokThreads);
    tokens_bwd_kernel<<<grid, kTokThreads, 0, stream>>>(
        reinterpret_cast<const uint4*>(dx0), reinterpret_cast<uint4*>(dpatch), reinterpret_cast<float4*>(dtok),
        static_cast<int>(B), T, static_cast<int>(N), static_cast<int>(P), D8);
    check_launch_tok("tokens_bwd");
}

}  // namespace b200
