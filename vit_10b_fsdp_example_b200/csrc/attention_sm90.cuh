// Device and host helpers shared by the attention kernels (attention_sm90.cu) and their attention-dropout
// instantiations (attention_drop_sm90.cu): tile configuration, TMA tile loads, the wgmma tile products, the kernel
// parameter blocks, the gradient-tile epilogue and the tensor-map set-up.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>

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

}  // namespace

}  // namespace b200
