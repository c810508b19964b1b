// The fused attention kernels for sm_90a, once: tile configuration, TMA tile loads, the wgmma tile products, the kernel
// parameter blocks, the attention-dropout mask, the forward and backward kernel bodies, the gradient-tile epilogue and
// the host-side launch.  Each body takes a compile-time kDrop: attention_sm90.cu instantiates the plain kernels
// (kDrop = false) and attention_drop_sm90.cu the attention-dropout ones (kDrop = true); see attention_sm90.cu for the
// algorithm and attention_drop_sm90.cu for the mask.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "dropout.cuh"
#include "gemm_sm90.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int kAttnThreads = 128;  // one warpgroup
constexpr int kTile = 64;          // rows of every Q / K / V / dO tile
constexpr float kLog2e = 1.4426950408889634f;

// hd-contiguous tiles use the widest swizzle atom that divides the tile width HD: 64 elements (SWIZZLE_128B), 32
// (SWIZZLE_64B) or 16 (SWIZZLE_32B).
template <int HD>
struct TileCfg {
    static constexpr int W = (HD % 64 == 0) ? 64 : (HD % 32 == 0) ? 32 : 16;
    static constexpr int kAtoms = HD / W;
    static constexpr int kRowBytes = W * 2;
    static constexpr uint32_t kMode = (W == 64) ? 1u : (W == 32) ? 2u : 3u;  // wgmma descriptor swizzle mode
    static constexpr int kAtomBytes = kTile * kRowBytes;
    static constexpr int kTileBytes = kTile * HD * 2;
    // Widths 64 / 128 / 160 are compiled for hd == HD.  The others read hd (HD - 16 < hd <= HD) at run time; TMA
    // zero-fills tile columns hd..HD-1, which add nothing to S or dP, and the epilogues store columns < hd only.
    static constexpr bool kFixedHd = HD == 64 || HD == 128 || HD == 160;
    static_assert(HD % 16 == 0 && HD <= 256, "unsupported tile width");
};

// Head dim served by the kernels of tile width HD.
template <int HD>
__device__ __forceinline__ int head_dim(int D, int H) { return TileCfg<HD>::kFixedHd ? HD : D / H; }

// One box per swizzle atom (W hd-columns x 64 rows); rows past the end of the image are zero-filled.
template <int HD>
__device__ __forceinline__ void load_tile(const CUtensorMap* tmap, uint64_t* bar, uint8_t* dst, int row0, int h, int b) {
    using T = TileCfg<HD>;
#pragma unroll
    for (int a = 0; a < T::kAtoms; ++a) tma_load_4d(tmap, bar, dst + a * T::kAtomBytes, a * T::W, row0, h, b);
}

// x[64 x 64] = A_tile (64 x hd) * B_tile (64 x hd)^T, both K-major in shared memory.
template <int HD>
__device__ __forceinline__ void mma_tile_nt(float (&x)[32], const uint8_t* sa, const uint8_t* sb) {
    using T = TileCfg<HD>;
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {
        const int atom = (k * 16) / T::W, within = (k * 16) % T::W;
        const uint32_t off = atom * T::kAtomBytes + within * 2;
        const uint64_t da = make_wgmma_desc(smem_u32(sa) + off, 0, 8 * T::kRowBytes, T::kMode);
        const uint64_t db = make_wgmma_desc(smem_u32(sb) + off, 0, 8 * T::kRowBytes, T::kMode);
        WgmmaSS<64, 0, 0>::mma(x, da, db, k > 0 ? 1u : 0u);
    }
}

// acc[64 x hd] += A (64 x 64, bf16 register fragments) * B_tile (64 x hd, MN-major: the 64 rows are the reduction).
template <int HD>
__device__ __forceinline__ void mma_tile_rs(float (&acc)[HD / 2], const uint32_t (&a)[4][4], const uint8_t* sb) {
    using T = TileCfg<HD>;
#pragma unroll
    for (int k = 0; k < kTile / 16; ++k) {
        // 8-row groups are 8*rowbytes apart (SBO), hd atoms are one tile-atom apart (LBO)
        const uint64_t db = make_wgmma_desc(smem_u32(sb) + k * 16 * T::kRowBytes, T::kAtomBytes, 8 * T::kRowBytes, T::kMode);
        WgmmaRS<HD, 1>::mma(acc, a[k], db, 1u);
    }
}

// fp32 accumulator tile (64 x 64) -> the four 16-wide-k A fragments of the next product.
__device__ __forceinline__ void pack_a_frags(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) a[c][i] = pack_bf16x2(x[8 * c + 2 * i], x[8 * c + 2 * i + 1]);
}

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

struct AttnParams {
    int N;             // tokens per image
    int H, B;
    int D;             // H * hd
    float scale_log2;  // hd^-1/2 * log2(e)
    float scale;       // hd^-1/2
    __nv_bfloat16* out;  // [B*N, D]
    float* lse;          // [B*H, N] or null
    __nv_bfloat16* p;    // [B*H, N, ldp] or null
    int64_t ldp;
};

struct BwdParams {
    int N, H, B, D;
    float scale_log2, scale;
    const float* lse;    // [B*H, N]
    const float* delta;  // [B*H, N]
    __nv_bfloat16* dqkv;  // [B*N, 3*D]
    float* colsum;        // [3*D] or null
};

struct DropParams {
    uint32_t key_lo, key_hi;
    uint32_t thresh16;  // keep <=> 16-bit chunk >= thresh16
    float scale;        // 1 / (1 - thresh16 / 65536)
};

// Keep bits of this thread's 32 tile elements when tile rows are queries (forward, dQ role); bit 4 * j + i belongs to
// x[4 * j + i] (i = 2 * row + column: rows r0 / r0 + 8, columns 8 j + cpair + 0 / 1).  A vector's 8 keys are spread
// over the 4 lanes of a quad; quad lane t evaluates both rows' vectors at column groups 2t and 2t + 1.
__device__ __forceinline__ uint32_t keep_bits_query_rows(const DropParams& d, int64_t bh, int N, int q0, int key0,
                                                         uint32_t lane) {
    const int64_t vecs = (N + 7) / 8;  // Philox vectors per probability row
    const uint32_t t = lane & 3;
    uint32_t own = 0;  // byte 2 * row + jj: vector (query q0 + 8 row, column group 2t + jj)
#pragma unroll
    for (int row = 0; row < 2; ++row)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
            own |= dropout_keep8((bh * N + q0 + 8 * row) * vecs + key0 / 8 + 2 * t + jj, d.key_lo, d.key_hi, d.thresh16)
                   << (8 * (2 * row + jj));
    uint32_t bits = 0;
#pragma unroll
    for (int src = 0; src < 4; ++src) {
        const uint32_t w = __shfl_sync(0xffffffffu, own, (lane & ~3u) | src) >> (2 * t);
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
            bits |= (((w >> (8 * jj)) & 3u) | (((w >> (8 * (2 + jj))) & 3u) << 2)) << (4 * (2 * src + jj));
    }
    return bits;
}

// The same when tile rows are keys and columns queries (dK/dV role): a vector's 8 keys are row r0 of the 8 lanes that
// share lane & 3 (one bit each; the warp's rows r0 / r0 + 8 lie in key groups kg0 / kg0 + 1).  Lane 4u + t evaluates
// the vectors of queries q0 + 8u + 2t + e (e = 0, 1) at both key groups.
__device__ __forceinline__ uint32_t keep_bits_key_rows(const DropParams& d, int64_t bh, int N, int kg0, int q0,
                                                       uint32_t lane) {
    const int64_t vecs = (N + 7) / 8;
    const uint32_t u = lane >> 2, t = lane & 3;
    uint32_t own = 0;  // byte 2 * g + e: vector (query q0 + 8u + 2t + e, key group kg0 + g)
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e)
            own |= dropout_keep8((bh * N + q0 + 8 * u + 2 * t + e) * vecs + kg0 + g, d.key_lo, d.key_hi, d.thresh16)
                   << (8 * (2 * g + e));
    uint32_t bits = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t w = __shfl_sync(0xffffffffu, own, 4 * j + t) >> u;  // this thread's keys are chunk u of a group
        bits |= ((w & 1u) | ((w >> 7) & 2u) | ((w >> 14) & 4u) | ((w >> 21) & 8u)) << (4 * j);
    }
    return bits;
}

__device__ __forceinline__ float keep_scale(uint32_t bits, int i, const DropParams& d) { return (bits >> i) & 1u ? d.scale : 0.f; }

// Barrier wait of the kernel bodies.  The dropout kernels wait without printf: a call in a wgmma kernel makes ptxas
// serialise its MMAs (C7510).  The plain kernels still use the printf wait.
template <bool kDrop>
__device__ __forceinline__ void attn_wait(uint64_t* bar, uint32_t phase) {
    if constexpr (kDrop) mbar_wait_silent(bar, phase);
    else mbar_wait(bar, phase);
}

// acc (64 x HD, rows = tokens of this tile) -> dqkv[token, col0 + :hd] and, optionally, its column sums.
template <int HD>
__device__ __forceinline__ void store_grad_tile(const float (&acc)[HD / 2], const BwdParams& p, int b, int row0, int r0,
                                                int cpair, int col0, uint32_t lane) {
    const int hd = head_dim<HD>(p.D, p.H);
    const int t0 = row0 + r0, t1 = t0 + 8;
    const bool ok0 = t0 < p.N, ok1 = t1 < p.N;
    __nv_bfloat16* g0 = p.dqkv + (static_cast<int64_t>(b) * p.N + t0) * (3 * p.D) + col0 + cpair;
    __nv_bfloat16* g1 = g0 + 8 * static_cast<int64_t>(3 * p.D);
#pragma unroll
    for (int j = 0; j < HD / 8; ++j) {
        if (j * 8 >= hd) continue;  // hd % 8 == 0: an 8-column group lies wholly inside or past the head
        const uint32_t w0 = ok0 ? pack_bf16x2(acc[4 * j], acc[4 * j + 1]) : 0u;
        const uint32_t w1 = ok1 ? pack_bf16x2(acc[4 * j + 2], acc[4 * j + 3]) : 0u;
        if (ok0) *reinterpret_cast<uint32_t*>(g0 + j * 8) = w0;
        if (ok1) *reinterpret_cast<uint32_t*>(g1 + j * 8) = w1;
        if (p.colsum != nullptr) {
            // bias gradient: sums of the bf16 values that were stored; the 8 lanes that share these columns reduce first
            float c0 = bf16_lo(w0) + bf16_lo(w1), c1 = bf16_hi(w0) + bf16_hi(w1);
#pragma unroll
            for (int sh = 4; sh < 32; sh <<= 1) {
                c0 += __shfl_xor_sync(0xffffffffu, c0, sh);
                c1 += __shfl_xor_sync(0xffffffffu, c1, sh);
            }
            if (lane < 4) {
                atomicAdd(p.colsum + col0 + j * 8 + cpair, c0);
                atomicAdd(p.colsum + col0 + j * 8 + cpair + 1, c1);
            }
        }
    }
}

// The kernel bodies take the parameter blocks by value and the dropout parameters as a pack d that is empty without
// dropout and one DropParams with it (kDrop).  Passed so, the plain and the dropout kernels compile to the same SASS as
// when each family had a kernel of its own; a reference, or a DropParams the plain kernels ignore, changes the SASS of
// the plain kernels (tests/test_attention_sass_unchanged.py).

// Forward of one work item.  With kDrop, P o M * s feeds O += P V while the row sums and the log-sum-exp stay those of
// the undropped P, and the probabilities are never written (p.p is null).
template <int HD, bool kDrop, typename... Drop>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k,
                                              const CUtensorMap& tmap_v, const AttnParams p, const Drop... d) {
    static_assert(sizeof...(Drop) == (kDrop ? 1 : 0), "one DropParams with dropout, none without");
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
        const int64_t bh = static_cast<int64_t>(b) * p.H + h;
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
        attn_wait<kDrop>(bar_q, ph_q);
        ph_q ^= 1;

        for (int kt = 0; kt < n_tiles; ++kt) {
            const int s = kt & 1;
            if (tid == 0 && kt + 1 < n_tiles) {  // the other slot was released by the barrier that ended tile kt - 1
                mbar_arrive_expect_tx(&bar_kv[s ^ 1], 2 * T::kTileBytes);
                load_tile<HD>(&tmap_k, &bar_kv[s ^ 1], sK + (s ^ 1) * T::kTileBytes, (kt + 1) * kTile, h, b);
                load_tile<HD>(&tmap_v, &bar_kv[s ^ 1], sV + (s ^ 1) * T::kTileBytes, (kt + 1) * kTile, h, b);
            }
            attn_wait<kDrop>(&bar_kv[s], (ph_kv >> s) & 1);
            ph_kv ^= 1u << s;

            float x[32];
            wgmma_fence();
            mma_tile_nt<HD>(x, sQ, sK + s * T::kTileBytes);
            wgmma_commit();
            uint32_t keep = 0;
            if constexpr (kDrop) keep = keep_bits_query_rows(d..., bh, p.N, qt * kTile + r0, kt * kTile, lane);  // MMAs run
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
            l0 = l0 * f0 + s0, l1 = l1 * f1 + s1;  // sums of the undropped probabilities
#pragma unroll
            for (int j = 0; j < HD / 8; ++j) {
                o[4 * j] *= f0, o[4 * j + 1] *= f0;
                o[4 * j + 2] *= f1, o[4 * j + 3] *= f1;
            }
            if constexpr (kDrop) {
#pragma unroll
                for (int i = 0; i < 32; ++i) x[i] *= keep_scale(keep, i, d...);
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
        // bh once more rather than the one above: the plain kernels keep their SASS only with it computed here
        const int64_t bh_out = static_cast<int64_t>(b) * p.H + h;
        __nv_bfloat16* orow0 = p.out + (static_cast<int64_t>(b) * p.N + q0) * p.D + h * hd + cpair;
        __nv_bfloat16* orow1 = orow0 + 8 * static_cast<int64_t>(p.D);
#pragma unroll
        for (int j = 0; j < HD / 8; ++j) {
            if (j * 8 >= hd) continue;  // zero-padded columns of the tile
            if (q0 < p.N) *reinterpret_cast<uint32_t*>(orow0 + j * 8) = pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
            if (q1 < p.N) *reinterpret_cast<uint32_t*>(orow1 + j * 8) = pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
        }
        if (p.lse != nullptr && (lane & 3) == 0) {
            if (q0 < p.N) p.lse[bh_out * p.N + q0] = m0 * p.scale + __logf(l0);
            if (q1 < p.N) p.lse[bh_out * p.N + q1] = m1 * p.scale + __logf(l1);
        }

        if constexpr (!kDrop) {
            if (p.p != nullptr) {
                // normalised probabilities for the un-fused backward: second pass over the keys with the final statistics
                const float lse0 = m0 * p.scale_log2 + __log2f(l0), lse1 = m1 * p.scale_log2 + __log2f(l1);
                __nv_bfloat16* prow0 = p.p + (bh_out * p.N + q0) * p.ldp;
                __nv_bfloat16* prow1 = prow0 + 8 * p.ldp;
                for (int kt = 0; kt < n_tiles; ++kt) {
                    if (tid == 0) {
                        mbar_arrive_expect_tx(&bar_kv[0], T::kTileBytes);
                        load_tile<HD>(&tmap_k, &bar_kv[0], sK, kt * kTile, h, b);
                    }
                    attn_wait<kDrop>(&bar_kv[0], ph_kv & 1);
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
}

// Backward of one work item.
// kRole 0: the CTA owns 64 keys (K, V tiles) and streams (Q, dO) tiles -> dK, dV.
// kRole 1: the CTA owns 64 queries (Q, dO tiles) and streams (K, V) tiles -> dQ.
// Either way x = own1 * str1^T is the score tile (transposed in role 0) and y = own2 * str2^T the dP tile.  With kDrop,
// dV += (P o M s)^T dO and dS = P o (dP o M s - delta).
template <int HD, int kRole, bool kDrop, typename... Drop>
__device__ __forceinline__ void attn_bwd_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k,
                                              const CUtensorMap& tmap_v, const CUtensorMap& tmap_do,
                                              const BwdParams p, const Drop... d) {
    static_assert(sizeof...(Drop) == (kDrop ? 1 : 0), "one DropParams with dropout, none without");
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
        attn_wait<kDrop>(bar_own, ph_own);
        ph_own ^= 1;

        for (int st = 0; st < n_tiles; ++st) {
            const int s = st & 1;
            if (tid == 0 && st + 1 < n_tiles) {
                mbar_arrive_expect_tx(&bar_str[s ^ 1], 2 * T::kTileBytes);
                load_tile<HD>(t_str1, &bar_str[s ^ 1], str1 + (s ^ 1) * T::kTileBytes, (st + 1) * kTile, h, b);
                load_tile<HD>(t_str2, &bar_str[s ^ 1], str2 + (s ^ 1) * T::kTileBytes, (st + 1) * kTile, h, b);
            }
            attn_wait<kDrop>(&bar_str[s], (ph_str >> s) & 1);
            ph_str ^= 1u << s;

            float x[32], y[32];
            wgmma_fence();
            mma_tile_nt<HD>(x, own1, str1 + s * T::kTileBytes);
            mma_tile_nt<HD>(y, own2, str2 + s * T::kTileBytes);
            wgmma_commit();
            // keep bits drawn while the MMAs run; role 0: rows r0 / r0 + 8 are keys in groups ot * 8 + 2 warp (+ 1)
            uint32_t keep = 0;
            if constexpr (kDrop)
                keep = kRole == 0
                           ? keep_bits_key_rows(d..., bh, p.N, ot * (kTile / 8) + 2 * static_cast<int>(warp), st * kTile, lane)
                           : keep_bits_query_rows(d..., bh, p.N, ot * kTile + r0, st * kTile, lane);
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
                float m0a = 1.f, m0b = 1.f, m1a = 1.f, m1b = 1.f;  // dropout mask times its scale
                if constexpr (kDrop) {
                    m0a = keep_scale(keep, 4 * j, d...), m0b = keep_scale(keep, 4 * j + 1, d...);
                    m1a = keep_scale(keep, 4 * j + 2, d...), m1b = keep_scale(keep, 4 * j + 3, d...);
                }
                x[4 * j] = p0a * m0a, x[4 * j + 1] = p0b * m0b, x[4 * j + 2] = p1a * m1a, x[4 * j + 3] = p1b * m1b;
                y[4 * j] = p0a * (y[4 * j] * m0a - d0a) * p.scale;
                y[4 * j + 1] = p0b * (y[4 * j + 1] * m0b - d0b) * p.scale;
                y[4 * j + 2] = p1a * (y[4 * j + 2] * m1a - d1a) * p.scale;
                y[4 * j + 3] = p1b * (y[4 * j + 3] * m1b - d1b) * p.scale;
            }
            uint32_t a[4][4];
            if constexpr (kRole == 0) {
                pack_a_frags(x, a);  // (P o M s)^T
                wgmma_fence();
                mma_tile_rs<HD>(acc1, a, str2 + s * T::kTileBytes);  // dV += (P o M s)^T dO
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

void check_launch(const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

template <typename Kern>
void set_smem(Kern kern, int bytes) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (err != cudaSuccess) throw std::runtime_error(std::string("attention smem attr: ") + cudaGetErrorString(err));
}

void qkv_operands(const __nv_bfloat16* qkv, int64_t ld_qkv, int N, int H, int hd, GemmOperand (&ops)[3]) {
    for (int i = 0; i < 3; ++i) {
        ops[i].ptr = qkv + static_cast<int64_t>(i) * H * hd;
        ops[i].ld = ld_qkv;
        ops[i].nb_inner = H, ops[i].stride_b_inner = hd;
        ops[i].nb_outer = 1, ops[i].stride_b_outer = 0;
    }
}

// Tensor map of one 64-row tile shape over a [B, N, H, hd] view (rows past N of an image and columns past hd of a
// head read as zeros).
template <int HD>
CUtensorMap tile_map(GemmOperand op, int B, int N, int hd) {
    op.nb_outer = B, op.stride_b_outer = static_cast<int64_t>(N) * op.ld;
    return make_tensor_map_4d(op, hd, N, TileCfg<HD>::W, kTile, TileCfg<HD>::kRowBytes);
}

// Tile width the kernels run head dim hd at (hd rounded up to 16), or 0 when they do not take hd.  hd % 8 == 0 because
// TMA needs the head stride (hd * 2 bytes) to be a multiple of 16.  hd = 56 / 120 / 152 would need zero-padded
// kernels at the widths 64 / 128 / 160, which are compiled for hd == width only.
constexpr int tile_width(int hd) {
    if (hd % 8 != 0 || hd < 32 || hd > 160) return 0;
    const int w = (hd + 15) / 16 * 16;
    return (w == 64 || w == 128 || w == 160) && w != hd ? 0 : w;
}

bool shape_ok(int N, int hd) { return N > 0 && N % 2 == 0 && tile_width(hd) != 0; }

// Calls f(std::integral_constant<int, W>) with the tile width W of hd; throws when no kernel takes hd.
template <typename F>
void dispatch_tile_width(int hd, const char* what, F&& f) {
    switch (tile_width(hd)) {
        case 32: return f(std::integral_constant<int, 32>());
        case 48: return f(std::integral_constant<int, 48>());
        case 64: return f(std::integral_constant<int, 64>());
        case 80: return f(std::integral_constant<int, 80>());
        case 96: return f(std::integral_constant<int, 96>());
        case 112: return f(std::integral_constant<int, 112>());
        case 128: return f(std::integral_constant<int, 128>());
        case 144: return f(std::integral_constant<int, 144>());
        case 160: return f(std::integral_constant<int, 160>());
    }
    throw std::runtime_error(std::string(what) + ": no kernel for head dim " + std::to_string(hd));
}

DropParams make_drop(float p, uint64_t key, const char* what) {
    if (!(p > 0.f && p < 1.f)) throw std::runtime_error(std::string(what) + ": dropout p must be in (0, 1)");
    DropParams d;
    d.key_lo = static_cast<uint32_t>(key), d.key_hi = static_cast<uint32_t>(key >> 32);
    d.thresh16 = dropout_thresh16(p);
    d.scale = dropout_scale(d.thresh16);
    return d;
}

// The kernels: thin wrappers around the bodies above, the plain ones defined in attention_sm90.cu and the dropout ones
// in attention_drop_sm90.cu.
template <int HD>
__global__ void attn_fwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                                     const __grid_constant__ CUtensorMap tmap_v, const AttnParams p);
template <int HD, int kRole>
__global__ void attn_bwd_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                                     const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                                     const BwdParams p);
template <int HD>
__global__ void attn_fwd_drop_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                          const __grid_constant__ CUtensorMap tmap_k,
                                          const __grid_constant__ CUtensorMap tmap_v, const AttnParams p,
                                          const DropParams d);
template <int HD, int kRole>
__global__ void attn_bwd_drop_sm90_kernel(const __grid_constant__ CUtensorMap tmap_q,
                                          const __grid_constant__ CUtensorMap tmap_k,
                                          const __grid_constant__ CUtensorMap tmap_v,
                                          const __grid_constant__ CUtensorMap tmap_do, const BwdParams p,
                                          const DropParams d);

template <int HD, bool kDrop>
void launch_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const AttnParams& p, const DropParams& d, cudaStream_t stream) {
    constexpr int kSmem = 5 * TileCfg<HD>::kTileBytes + 64;
    GemmOperand ops[3];
    const int hd = p.D / p.H;
    qkv_operands(qkv, ld_qkv, p.N, p.H, hd, ops);
    const CUtensorMap tq = tile_map<HD>(ops[0], p.B, p.N, hd), tk = tile_map<HD>(ops[1], p.B, p.N, hd),
                      tv = tile_map<HD>(ops[2], p.B, p.N, hd);
    const int items = (p.N + kTile - 1) / kTile * p.H * p.B;
    static bool attr_set = false;
    if constexpr (kDrop) {
        auto kern = attn_fwd_drop_sm90_kernel<HD>;
        if (!attr_set) set_smem(kern, kSmem), attr_set = true;
        kern<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, p, d);
        check_launch("attention forward (dropout) launch");
    } else {
        auto kern = attn_fwd_sm90_kernel<HD>;
        if (!attr_set) set_smem(kern, kSmem), attr_set = true;
        kern<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, p);
        check_launch("attention forward launch");
    }
}

template <int HD, bool kDrop>
void launch_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do, const BwdParams& p,
                const DropParams& d, cudaStream_t stream) {
    constexpr int kSmem = 6 * TileCfg<HD>::kTileBytes + 64;
    GemmOperand ops[3], od;
    const int hd = p.D / p.H;
    qkv_operands(qkv, ld_qkv, p.N, p.H, hd, ops);
    od.ptr = dout, od.ld = ld_do, od.nb_inner = p.H, od.stride_b_inner = hd;
    const CUtensorMap tq = tile_map<HD>(ops[0], p.B, p.N, hd), tk = tile_map<HD>(ops[1], p.B, p.N, hd),
                      tv = tile_map<HD>(ops[2], p.B, p.N, hd), tdo = tile_map<HD>(od, p.B, p.N, hd);
    const int items = (p.N + kTile - 1) / kTile * p.H * p.B;
    static bool attr_set = false;
    if constexpr (kDrop) {
        auto kern_kv = attn_bwd_drop_sm90_kernel<HD, 0>;
        auto kern_q = attn_bwd_drop_sm90_kernel<HD, 1>;
        if (!attr_set) set_smem(kern_kv, kSmem), set_smem(kern_q, kSmem), attr_set = true;
        kern_kv<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p, d);
        check_launch("attention backward (dK/dV, dropout) launch");
        kern_q<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p, d);
        check_launch("attention backward (dQ, dropout) launch");
    } else {
        auto kern_kv = attn_bwd_sm90_kernel<HD, 0>;
        auto kern_q = attn_bwd_sm90_kernel<HD, 1>;
        if (!attr_set) set_smem(kern_kv, kSmem), set_smem(kern_q, kSmem), attr_set = true;
        kern_kv<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p);
        check_launch("attention backward (dK/dV) launch");
        kern_q<<<items, kAttnThreads, kSmem, stream>>>(tq, tk, tv, tdo, p);
        check_launch("attention backward (dQ) launch");
    }
}

// Forward / backward at hd's tile width, without (kDrop = false, d unused) or with attention dropout.
template <bool kDrop>
void run_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, __nv_bfloat16* probs,
             int64_t ldp, int B, int N, int H, int hd, const DropParams& d, cudaStream_t stream) {
    AttnParams p;
    p.N = N, p.H = H, p.B = B, p.D = H * hd;
    p.scale = 1.0f / sqrtf(static_cast<float>(hd));
    p.scale_log2 = p.scale * kLog2e;
    p.out = out, p.lse = lse, p.p = probs, p.ldp = ldp;
    dispatch_tile_width(hd, "attention_fwd",
                        [&](auto w) { launch_fwd<decltype(w)::value, kDrop>(qkv, ld_qkv, p, d, stream); });
}

template <bool kDrop>
void run_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do, const float* lse,
             const float* delta, __nv_bfloat16* dqkv, int B, int N, int H, int hd, float* colsum, const DropParams& d,
             cudaStream_t stream) {
    BwdParams p;
    p.N = N, p.H = H, p.B = B, p.D = H * hd;
    p.scale = 1.0f / sqrtf(static_cast<float>(hd));
    p.scale_log2 = p.scale * kLog2e;
    p.lse = lse, p.delta = delta, p.dqkv = dqkv, p.colsum = colsum;
    dispatch_tile_width(hd, "attention_bwd",
                        [&](auto w) { launch_bwd<decltype(w)::value, kDrop>(qkv, ld_qkv, dout, ld_do, p, d, stream); });
}

}  // namespace

}  // namespace b200
