// Fused multi-head attention for sm_90a: softmax(Q K^T * hd^-1/2) V and its backward, flash style (scores never
// reach HBM), for any even sequence length and every head dim hd with hd % 8 == 0 and 32 <= hd <= 160 except 56 / 120 /
// 152.  Tiles are W = hd rounded up to 16 columns wide; the widths 64 / 128 / 160 are compiled for hd == W, the widths
// 32 / 48 / 80 / 96 / 112 / 144 read hd at run time and TMA zero-fills the tile columns past it (attention_sm90.cuh).
//
//   TMA     : 64-row tiles of Q / K / V / dO are read *in place* from the packed qkv activation ([tokens, 3*D], head h
//             of q at columns h*hd) through 4-D tensor maps -- no permute / split copies.  Streamed tiles are double
//             buffered: the next tile's loads fly while the current one is computed.
//   wgmma   : one warpgroup per CTA.  S = Q K^T (m64n64k16, both operands from swizzled shared memory, fp32
//             accumulators in registers); the bf16-packed probabilities are fed back as the *register* A operand of
//             O += P V, with V consumed as an MN-major operand (no transpose, no round trip through shared memory).
//   softmax : online (running max / sum per query row, exp2 with the scale folded in); a thread owns two rows of the
//             tile, the four lanes that share a row reduce with shuffles.
//   forward : O [tokens, D] bf16, log-sum-exp per row (fp32), optionally the normalised probabilities P (a second
//             pass over the keys; only the un-fused backward needs them).
//   backward: delta = rowsum(dO o O), then one kernel in two roles.  Role 0 owns a 64-key tile and streams (Q, dO):
//             S^T = K Q^T, dP^T = V dO^T, dV += P^T dO, dK += dS^T Q.  Role 1 owns a 64-query tile and streams (K, V):
//             dQ += dS K.  P is rebuilt from the stored log-sum-exp; no atomics on the gradients.  The qkv bias
//             gradient (column sums of dq | dk | dv) is reduced from the bf16-rounded tiles in the epilogue.
//   dropout : attention_fwd / attention_bwd with drop_p > 0 run the attention-dropout kernels (attention_drop_sm90.cu).
//
// The kernel bodies and the launch code are in attention_sm90.cuh, shared with the dropout kernels through a
// compile-time kDrop; this file holds the plain kernels (kDrop = false), the delta kernel and the host entry points.
//
// A work item is one (image, head, 64-row tile) and gets one CTA.  (A persistent grid of resident CTAs looping over
// items was measured too: within 2 % at hd = 160 and 25 % slower in the backward at hd = 64, ViT-L shape, H100 80GB
// HBM3 at 700 W, so it is not offered.)  Status: a first Hopper version -- a single warpgroup waits for every wgmma
// batch before it goes on, so softmax and tensor-core work of one CTA do not overlap, and the hd = 160 dK/dV role
// sits at the 255-register limit with a few spilled bytes.  Replaces timm Attention's materialised [B,H,N,N] softmax (reference
// run_vit_training.py:134 -> timm Block -> Attention) and its autograd backward.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

#include "attention_sm90.h"
#include "attention_sm90.cuh"

namespace b200 {

namespace {

template <int HD>
__global__ void __launch_bounds__(kAttnThreads) attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                                                    const __grid_constant__ CUtensorMap tmap_k,
                                                                    const __grid_constant__ CUtensorMap tmap_v,
                                                                    const AttnParams p) {
    attn_fwd_body<HD, false>(tmap_q, tmap_k, tmap_v, p);
}

template <int HD, int kRole>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                                                    const __grid_constant__ CUtensorMap tmap_k,
                                                                    const __grid_constant__ CUtensorMap tmap_v,
                                                                    const __grid_constant__ CUtensorMap tmap_do,
                                                                    const BwdParams p) {
    attn_bwd_body<HD, kRole, false>(tmap_q, tmap_k, tmap_v, tmap_do, p);
}

// delta[b*H + h, q] = sum_d dO[b*N + q, h*hd + d] * O[b*N + q, h*hd + d]; one warp per (token, head).
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, int64_t ld_do, const __nv_bfloat16* __restrict__ out,
                                  int64_t ld_o, float* __restrict__ delta, int B, int N, int H, int hd) {
    const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x & 31;
    if (w >= static_cast<int64_t>(B) * N * H) return;
    const int h = static_cast<int>(w % H);
    const int64_t tok = w / H;
    const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(dout + tok * ld_do + h * hd);
    const __nv_bfloat162* o = reinterpret_cast<const __nv_bfloat162*>(out + tok * ld_o + h * hd);
    float s = 0.f;
    for (int i = lane; i < hd / 2; i += 32) {
        const float2 x = __bfloat1622float2(a[i]), y = __bfloat1622float2(o[i]);
        s += x.x * y.x + x.y * y.y;
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) s += __shfl_xor_sync(0xffffffffu, s, sh);
    if (lane == 0) delta[(tok / N * H + h) * N + tok % N] = s;
}

}  // namespace

// The model's routing (cuda_ops.use_flash): the kernels take every head dim shape_ok accepts, but a new tile width is
// routed only where the fused pair beats the un-fused route (which keeps P) in the forward *and* the backward without
// dropout.  tools/bench_attention.py, B128 N256 H16, H100 80GB HBM3 at 700 W, medians of 20, three runs, backward
// fused / un-fused: hd 32 / 40 / 48 take 0.51 / 0.76 / 0.65 times the un-fused time, so widths 32 and 48 are routed.
// hd 72 / 80 (W 80) take 1.11 / 1.02 times, hd 88 / 96 (W 96) 1.11 / 1.00, hd 104 / 112 (W 112) 1.34 / 1.20 and
// hd 136 / 144 (W 144) 1.30 / 1.17, so those widths stay un-fused by default.  64 / 128 / 160 keep their route.
bool attention_supported(int N, int hd) {
    return shape_ok(N, hd) && (hd == 64 || hd == 128 || hd == 160 || tile_width(hd) <= 48);
}

bool attention_shape_ok(int N, int hd) { return shape_ok(N, hd); }

void attention_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, __nv_bfloat16* probs,
                   int64_t ldp, int B, int N, int H, int hd, cudaStream_t stream, float drop_p, uint64_t drop_key) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_fwd: unsupported (N, head_dim)");
    if (drop_p != 0.f) {
        if (probs != nullptr) throw std::runtime_error("attention_fwd: no probability output with dropout");
        attention_fwd_drop(qkv, ld_qkv, out, lse, B, N, H, hd, drop_p, drop_key, stream);
        return;
    }
    run_fwd<false>(qkv, ld_qkv, out, lse, probs, ldp, B, N, H, hd, DropParams{}, stream);
}

void attention_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                   const __nv_bfloat16* out, int64_t ld_o, const float* lse, float* delta, __nv_bfloat16* dqkv,
                   int B, int N, int H, int hd, cudaStream_t stream, float* colsum, float drop_p, uint64_t drop_key) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_bwd: unsupported (N, head_dim)");
    if (drop_p != 0.f) make_drop(drop_p, drop_key, "attention_bwd");  // a bad p throws before the delta kernel runs
    const int64_t warps = static_cast<int64_t>(B) * N * H;
    attn_delta_kernel<<<static_cast<unsigned>((warps + 7) / 8), 256, 0, stream>>>(dout, ld_do, out, ld_o, delta, B, N, H, hd);
    check_launch("attention delta launch");
    if (drop_p != 0.f) {
        attention_bwd_drop(qkv, ld_qkv, dout, ld_do, lse, delta, dqkv, B, N, H, hd, colsum, drop_p, drop_key, stream);
        return;
    }
    run_bwd<false>(qkv, ld_qkv, dout, ld_do, lse, delta, dqkv, B, N, H, hd, colsum, DropParams{}, stream);
}

}  // namespace b200
