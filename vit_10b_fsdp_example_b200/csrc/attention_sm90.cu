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
//   dropout : attention_fwd / attention_bwd with drop_p > 0 run the attention-dropout instantiations of these kernels
//             (attention_drop_sm90.cu); the helpers both files use are in attention_sm90.cuh.
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
    using T = TileCfg<HD>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + T::kTileBytes;      // [2]
    uint8_t* sV = sK + 2 * T::kTileBytes;  // [2]
    uint64_t* bar_q = reinterpret_cast<uint64_t*>(sV + 2 * T::kTileBytes);
    uint64_t* bar_kv = bar_q + 1;          // [2]

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int r0 = warp * 16 + lane / 4;   // this thread's rows of the tile: r0 and r0 + 8
    const int cpair = (lane & 3) * 2;      // its two adjacent columns inside every 8-column group

    if (tid == 0) {
        prefetch_tmap(&tmap_q);
        prefetch_tmap(&tmap_k);
        prefetch_tmap(&tmap_v);
        mbar_init(bar_q, 1);
        mbar_init(&bar_kv[0], 1);
        mbar_init(&bar_kv[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    const int n_tiles = (p.N + kTile - 1) / kTile;
    const int total = n_tiles * p.H * p.B;
    uint32_t ph_q = 0, ph_kv = 0;  // bit s of ph_kv = parity the next wait on bar_kv[s] uses

    if (const int item = blockIdx.x; item < total) {  // one CTA per work item
        const int qt = item % n_tiles, h = (item / n_tiles) % p.H, b = item / (n_tiles * p.H);
        if (tid == 0) {
            mbar_arrive_expect_tx(bar_q, T::kTileBytes);
            load_tile<HD>(&tmap_q, bar_q, sQ, qt * kTile, h, b);
            mbar_arrive_expect_tx(&bar_kv[0], 2 * T::kTileBytes);
            load_tile<HD>(&tmap_k, &bar_kv[0], sK, 0, h, b);
            load_tile<HD>(&tmap_v, &bar_kv[0], sV, 0, h, b);
        }
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // running max (raw scores) / partial sums per row
        mbar_wait(bar_q, ph_q);
        ph_q ^= 1;

        for (int kt = 0; kt < n_tiles; ++kt) {
            const int s = kt & 1;
            if (tid == 0 && kt + 1 < n_tiles) {  // the other slot was released by the barrier that ended tile kt - 1
                mbar_arrive_expect_tx(&bar_kv[s ^ 1], 2 * T::kTileBytes);
                load_tile<HD>(&tmap_k, &bar_kv[s ^ 1], sK + (s ^ 1) * T::kTileBytes, (kt + 1) * kTile, h, b);
                load_tile<HD>(&tmap_v, &bar_kv[s ^ 1], sV + (s ^ 1) * T::kTileBytes, (kt + 1) * kTile, h, b);
            }
            mbar_wait(&bar_kv[s], (ph_kv >> s) & 1);
            ph_kv ^= 1u << s;

            float x[32];
            wgmma_fence();
            mma_tile_nt<HD>(x, sQ, sK + s * T::kTileBytes);
            wgmma_commit();
            wgmma_wait<0>();

            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int key = kt * kTile + j * 8 + cpair;
                if (key >= p.N) x[4 * j] = x[4 * j + 2] = -INFINITY;
                if (key + 1 >= p.N) x[4 * j + 1] = x[4 * j + 3] = -INFINITY;
                mx0 = fmaxf(mx0, fmaxf(x[4 * j], x[4 * j + 1]));
                mx1 = fmaxf(mx1, fmaxf(x[4 * j + 2], x[4 * j + 3]));
            }
            const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
            const float f0 = exp2f((m0 - mn0) * p.scale_log2), f1 = exp2f((m1 - mn1) * p.scale_log2);
            m0 = mn0, m1 = mn1;
            const float ms0 = mn0 * p.scale_log2, ms1 = mn1 * p.scale_log2;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                x[4 * j] = exp2f(fmaf(x[4 * j], p.scale_log2, -ms0));
                x[4 * j + 1] = exp2f(fmaf(x[4 * j + 1], p.scale_log2, -ms0));
                x[4 * j + 2] = exp2f(fmaf(x[4 * j + 2], p.scale_log2, -ms1));
                x[4 * j + 3] = exp2f(fmaf(x[4 * j + 3], p.scale_log2, -ms1));
                s0 += x[4 * j] + x[4 * j + 1];
                s1 += x[4 * j + 2] + x[4 * j + 3];
            }
            l0 = l0 * f0 + s0, l1 = l1 * f1 + s1;
#pragma unroll
            for (int j = 0; j < HD / 8; ++j) {
                o[4 * j] *= f0, o[4 * j + 1] *= f0;
                o[4 * j + 2] *= f1, o[4 * j + 3] *= f1;
            }
            uint32_t a[4][4];
            pack_a_frags(x, a);
            wgmma_fence();
            mma_tile_rs<HD>(o, a, sV + s * T::kTileBytes);
            wgmma_commit();
            wgmma_wait<0>();
            __syncthreads();  // every warp is done with slot s (and, after the last tile, with Q)
        }

        // ---- epilogue: O / sum -> bf16 -> out[token, h*hd + :] ----
        l0 = quad_sum(l0), l1 = quad_sum(l1);
        const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
        const int q0 = qt * kTile + r0, q1 = q0 + 8;
        const int hd = head_dim<HD>(p.D, p.H);
        const int64_t bh = static_cast<int64_t>(b) * p.H + h;
        __nv_bfloat16* orow0 = p.out + (static_cast<int64_t>(b) * p.N + q0) * p.D + h * hd + cpair;
        __nv_bfloat16* orow1 = orow0 + 8 * static_cast<int64_t>(p.D);
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
            if (j * 8 >= hd) continue;  // zero-padded columns of the tile
            if (q0 < p.N) *reinterpret_cast<uint32_t*>(orow0 + j * 8) = pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
            if (q1 < p.N) *reinterpret_cast<uint32_t*>(orow1 + j * 8) = pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
        }
        if (p.lse != nullptr && (lane & 3) == 0) {
            if (q0 < p.N) p.lse[bh * p.N + q0] = m0 * p.scale + __logf(l0);
            if (q1 < p.N) p.lse[bh * p.N + q1] = m1 * p.scale + __logf(l1);
        }

        if (p.p != nullptr) {
            // normalised probabilities for the un-fused backward: second pass over the keys with the final statistics
            const float lse0 = m0 * p.scale_log2 + __log2f(l0), lse1 = m1 * p.scale_log2 + __log2f(l1);
            __nv_bfloat16* prow0 = p.p + (bh * p.N + q0) * p.ldp;
            __nv_bfloat16* prow1 = prow0 + 8 * p.ldp;
            for (int kt = 0; kt < n_tiles; ++kt) {
                if (tid == 0) {
                    mbar_arrive_expect_tx(&bar_kv[0], T::kTileBytes);
                    load_tile<HD>(&tmap_k, &bar_kv[0], sK, kt * kTile, h, b);
                }
                mbar_wait(&bar_kv[0], ph_kv & 1);
                ph_kv ^= 1u;
                float x[32];
                wgmma_fence();
                mma_tile_nt<HD>(x, sQ, sK);
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int key = kt * kTile + j * 8 + cpair;
                    if (key >= p.N) continue;  // N is even: key + 1 is valid too
                    if (q0 < p.N)
                        *reinterpret_cast<uint32_t*>(prow0 + key) =
                            pack_bf16x2(exp2f(fmaf(x[4 * j], p.scale_log2, -lse0)), exp2f(fmaf(x[4 * j + 1], p.scale_log2, -lse0)));
                    if (q1 < p.N)
                        *reinterpret_cast<uint32_t*>(prow1 + key) =
                            pack_bf16x2(exp2f(fmaf(x[4 * j + 2], p.scale_log2, -lse1)), exp2f(fmaf(x[4 * j + 3], p.scale_log2, -lse1)));
                }
                __syncthreads();
            }
        }
    }
}

// kRole 0: the CTA owns 64 keys (K, V tiles) and streams (Q, dO) tiles -> dK, dV.
// kRole 1: the CTA owns 64 queries (Q, dO tiles) and streams (K, V) tiles -> dQ.
// Either way x = own1 * str1^T is the score tile (transposed in role 0) and y = own2 * str2^T the dP tile.
template <int HD, int kRole>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                                                    const __grid_constant__ CUtensorMap tmap_k,
                                                                    const __grid_constant__ CUtensorMap tmap_v,
                                                                    const __grid_constant__ CUtensorMap tmap_do,
                                                                    const BwdParams p) {
    using T = TileCfg<HD>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* own1 = smem;
    uint8_t* own2 = own1 + T::kTileBytes;
    uint8_t* str1 = own2 + T::kTileBytes;      // [2]
    uint8_t* str2 = str1 + 2 * T::kTileBytes;  // [2]
    uint64_t* bar_own = reinterpret_cast<uint64_t*>(str2 + 2 * T::kTileBytes);
    uint64_t* bar_str = bar_own + 1;           // [2]
    const CUtensorMap* t_own1 = kRole == 0 ? &tmap_k : &tmap_q;
    const CUtensorMap* t_own2 = kRole == 0 ? &tmap_v : &tmap_do;
    const CUtensorMap* t_str1 = kRole == 0 ? &tmap_q : &tmap_k;
    const CUtensorMap* t_str2 = kRole == 0 ? &tmap_do : &tmap_v;

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int r0 = warp * 16 + lane / 4;
    const int cpair = (lane & 3) * 2;

    if (tid == 0) {
        prefetch_tmap(&tmap_q);
        prefetch_tmap(&tmap_k);
        prefetch_tmap(&tmap_v);
        prefetch_tmap(&tmap_do);
        mbar_init(bar_own, 1);
        mbar_init(&bar_str[0], 1);
        mbar_init(&bar_str[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    const int n_tiles = (p.N + kTile - 1) / kTile;
    const int total = n_tiles * p.H * p.B;
    uint32_t ph_own = 0, ph_str = 0;

    if (const int item = blockIdx.x; item < total) {  // one CTA per work item
        const int ot = item % n_tiles, h = (item / n_tiles) % p.H, b = item / (n_tiles * p.H);
        const int64_t bh = static_cast<int64_t>(b) * p.H + h;
        const float* lse = p.lse + bh * p.N;
        const float* delta = p.delta + bh * p.N;
        if (tid == 0) {
            mbar_arrive_expect_tx(bar_own, 2 * T::kTileBytes);
            load_tile<HD>(t_own1, bar_own, own1, ot * kTile, h, b);
            load_tile<HD>(t_own2, bar_own, own2, ot * kTile, h, b);
            mbar_arrive_expect_tx(&bar_str[0], 2 * T::kTileBytes);
            load_tile<HD>(t_str1, &bar_str[0], str1, 0, h, b);
            load_tile<HD>(t_str2, &bar_str[0], str2, 0, h, b);
        }
        float acc1[HD / 2];                      // dV (role 0) or dQ (role 1)
        float acc2[kRole == 0 ? HD / 2 : 1];     // dK (role 0)
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) acc1[i] = 0.f;
#pragma unroll
        for (int i = 0; i < (kRole == 0 ? HD / 2 : 1); ++i) acc2[i] = 0.f;
        // role 1: the statistics belong to this thread's two query rows
        float rl0 = 0.f, rl1 = 0.f, rd0 = 0.f, rd1 = 0.f;
        if (kRole == 1) {
            const int q0 = ot * kTile + r0, q1 = q0 + 8;
            if (q0 < p.N) rl0 = lse[q0] * kLog2e, rd0 = delta[q0];
            if (q1 < p.N) rl1 = lse[q1] * kLog2e, rd1 = delta[q1];
        }
        mbar_wait(bar_own, ph_own);
        ph_own ^= 1;

        for (int st = 0; st < n_tiles; ++st) {
            const int s = st & 1;
            if (tid == 0 && st + 1 < n_tiles) {
                mbar_arrive_expect_tx(&bar_str[s ^ 1], 2 * T::kTileBytes);
                load_tile<HD>(t_str1, &bar_str[s ^ 1], str1 + (s ^ 1) * T::kTileBytes, (st + 1) * kTile, h, b);
                load_tile<HD>(t_str2, &bar_str[s ^ 1], str2 + (s ^ 1) * T::kTileBytes, (st + 1) * kTile, h, b);
            }
            mbar_wait(&bar_str[s], (ph_str >> s) & 1);
            ph_str ^= 1u << s;

            float x[32], y[32];
            wgmma_fence();
            mma_tile_nt<HD>(x, own1, str1 + s * T::kTileBytes);
            mma_tile_nt<HD>(y, own2, str2 + s * T::kTileBytes);
            wgmma_commit();
            wgmma_wait<0>();

            const int row_tok0 = ot * kTile + r0, row_tok1 = row_tok0 + 8;  // tokens of this thread's rows
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col_tok = st * kTile + j * 8 + cpair;             // token of the first of its two columns
                const bool cok = col_tok < p.N;                             // N is even: col_tok + 1 is valid too
                float l0a, l0b, l1a, l1b, d0a, d0b, d1a, d1b;                // (row 0 | 1, column a | b)
                if (kRole == 0) {  // statistics follow the query = column
                    float2 lv = make_float2(0.f, 0.f), dv = make_float2(0.f, 0.f);
                    if (cok) {
                        lv = __ldg(reinterpret_cast<const float2*>(lse + col_tok));
                        dv = __ldg(reinterpret_cast<const float2*>(delta + col_tok));
                    }
                    l0a = l1a = lv.x * kLog2e, l0b = l1b = lv.y * kLog2e;
                    d0a = d1a = dv.x, d0b = d1b = dv.y;
                } else {
                    l0a = l0b = rl0, l1a = l1b = rl1;
                    d0a = d0b = rd0, d1a = d1b = rd1;
                }
                const bool ok0 = cok && row_tok0 < p.N, ok1 = cok && row_tok1 < p.N;
                const float p0a = ok0 ? exp2f(fmaf(x[4 * j], p.scale_log2, -l0a)) : 0.f;
                const float p0b = ok0 ? exp2f(fmaf(x[4 * j + 1], p.scale_log2, -l0b)) : 0.f;
                const float p1a = ok1 ? exp2f(fmaf(x[4 * j + 2], p.scale_log2, -l1a)) : 0.f;
                const float p1b = ok1 ? exp2f(fmaf(x[4 * j + 3], p.scale_log2, -l1b)) : 0.f;
                x[4 * j] = p0a, x[4 * j + 1] = p0b, x[4 * j + 2] = p1a, x[4 * j + 3] = p1b;
                y[4 * j] = p0a * (y[4 * j] - d0a) * p.scale;
                y[4 * j + 1] = p0b * (y[4 * j + 1] - d0b) * p.scale;
                y[4 * j + 2] = p1a * (y[4 * j + 2] - d1a) * p.scale;
                y[4 * j + 3] = p1b * (y[4 * j + 3] - d1b) * p.scale;
            }
            uint32_t a[4][4];
            if constexpr (kRole == 0) {
                pack_a_frags(x, a);  // P^T
                wgmma_fence();
                mma_tile_rs<HD>(acc1, a, str2 + s * T::kTileBytes);  // dV += P^T dO
                wgmma_commit();
                wgmma_wait<0>();
                pack_a_frags(y, a);  // dS^T
                wgmma_fence();
                mma_tile_rs<HD>(acc2, a, str1 + s * T::kTileBytes);  // dK += dS^T Q
            } else {
                pack_a_frags(y, a);  // dS
                wgmma_fence();
                mma_tile_rs<HD>(acc1, a, str1 + s * T::kTileBytes);  // dQ += dS K
            }
            wgmma_commit();
            wgmma_wait<0>();
            __syncthreads();  // every warp is done with slot s (and, after the last tile, with the owned tiles)
        }

        const int hd = head_dim<HD>(p.D, p.H);
        if constexpr (kRole == 0) {
            store_grad_tile<HD>(acc2, p, b, ot * kTile, r0, cpair, p.D + h * hd, lane);
            store_grad_tile<HD>(acc1, p, b, ot * kTile, r0, cpair, 2 * p.D + h * hd, lane);
        } else {
            store_grad_tile<HD>(acc1, p, b, ot * kTile, r0, cpair, h * hd, lane);
        }
    }
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

template <int HD>
void launch_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const AttnParams& p, cudaStream_t stream) {
    constexpr int kSmem = 5 * TileCfg<HD>::kTileBytes + 64;
    auto kern = attn_fwd_sm90_kernel<HD>;
    static bool attr_set = false;
    if (!attr_set) set_smem(kern, kSmem), attr_set = true;
    GemmOperand ops[3];
    const int hd = p.D / p.H;
    qkv_operands(qkv, ld_qkv, p.N, p.H, hd, ops);
    const CUtensorMap tq = tile_map<HD>(ops[0], p.B, p.N, hd), tk = tile_map<HD>(ops[1], p.B, p.N, hd),
                      tv = tile_map<HD>(ops[2], p.B, p.N, hd);
    const int items = (p.N + kTile - 1) / kTile * p.H * p.B;
    kern<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, p);
    check_launch("attention forward launch");
}

template <int HD>
void launch_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do, const BwdParams& p,
                cudaStream_t stream) {
    constexpr int kSmem = 6 * TileCfg<HD>::kTileBytes + 64;
    auto kern_kv = attn_bwd_sm90_kernel<HD, 0>;
    auto kern_q = attn_bwd_sm90_kernel<HD, 1>;
    static bool attr_set = false;
    if (!attr_set) set_smem(kern_kv, kSmem), set_smem(kern_q, kSmem), attr_set = true;
    GemmOperand ops[3], od;
    const int hd = p.D / p.H;
    qkv_operands(qkv, ld_qkv, p.N, p.H, hd, ops);
    od.ptr = dout, od.ld = ld_do, od.nb_inner = p.H, od.stride_b_inner = hd;
    const CUtensorMap tq = tile_map<HD>(ops[0], p.B, p.N, hd), tk = tile_map<HD>(ops[1], p.B, p.N, hd),
                      tv = tile_map<HD>(ops[2], p.B, p.N, hd), tdo = tile_map<HD>(od, p.B, p.N, hd);
    const int items = (p.N + kTile - 1) / kTile * p.H * p.B;
    kern_kv<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p);
    check_launch("attention backward (dK/dV) launch");
    kern_q<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p);
    check_launch("attention backward (dQ) launch");
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

void attention_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, __nv_bfloat16* probs,
                   int64_t ldp, int B, int N, int H, int hd, cudaStream_t stream, float drop_p, uint64_t drop_key) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_fwd: unsupported (N, head_dim)");
    if (drop_p != 0.f) {
        if (probs != nullptr) throw std::runtime_error("attention_fwd: no probability output with dropout");
        attention_fwd_drop(qkv, ld_qkv, out, lse, B, N, H, hd, drop_p, drop_key, stream);
        return;
    }
    AttnParams p;
    p.N = N, p.H = H, p.B = B, p.D = H * hd;
    p.scale = 1.0f / sqrtf(static_cast<float>(hd));
    p.scale_log2 = p.scale * kLog2e;
    p.out = out, p.lse = lse, p.p = probs, p.ldp = ldp;
    dispatch_tile_width(hd, "attention_fwd", [&](auto w) { launch_fwd<decltype(w)::value>(qkv, ld_qkv, p, stream); });
}

void attention_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                   const __nv_bfloat16* out, int64_t ld_o, const float* lse, float* delta, __nv_bfloat16* dqkv,
                   int B, int N, int H, int hd, cudaStream_t stream, float* colsum, float drop_p, uint64_t drop_key) {
    if (!shape_ok(N, hd)) throw std::runtime_error("attention_bwd: unsupported (N, head_dim)");
    const int64_t warps = static_cast<int64_t>(B) * N * H;
    attn_delta_kernel<<<static_cast<unsigned>((warps + 7) / 8), 256, 0, stream>>>(dout, ld_do, out, ld_o, delta, B, N, H, hd);
    check_launch("attention delta launch");
    if (drop_p != 0.f) {
        attention_bwd_drop(qkv, ld_qkv, dout, ld_do, lse, delta, dqkv, B, N, H, hd, colsum, drop_p, drop_key, stream);
        return;
    }
    BwdParams p;
    p.N = N, p.H = H, p.B = B, p.D = H * hd;
    p.scale = 1.0f / sqrtf(static_cast<float>(hd));
    p.scale_log2 = p.scale * kLog2e;
    p.lse = lse, p.delta = delta, p.dqkv = dqkv, p.colsum = colsum;
    dispatch_tile_width(hd, "attention_bwd",
                        [&](auto w) { launch_bwd<decltype(w)::value>(qkv, ld_qkv, dout, ld_do, p, stream); });
}

}  // namespace b200
