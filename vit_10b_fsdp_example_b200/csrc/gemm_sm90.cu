// Persistent, warp-specialised bf16 GEMM for sm_90a (H100):
//   TMA (cp.async.bulk.tensor, SWIZZLE_128B)  ->  shared-memory ring (mbarrier full / empty pairs)
//   wgmma.mma_async m64 x BLOCK_N x 16, two consumer warpgroups per CTA, fp32 accumulators in registers
//   fused epilogue (bias, exact GELU, dGELU, SwiGLU, dSwiGLU, per-row scale, residual add, pre-activation side
//   output, bias-gradient column sums)  ->  swizzled smem  ->  TMA store.
//
// One CTA owns a 128 x BLOCK_N output tile; a producer warp (with a reduced register budget) keeps the ring
// full while the consumer warpgroups (each 64 rows of the tile) issue the MMAs and run the epilogue.
//
//   D[b][m, n] = epilogue( sum_k A[b][m, k] * B[b][n, k] )
//
// A and B may each be K-major (reduction dim contiguous) or MN-major (reduction dim strided), which
// covers forward (NT), dgrad (NN) and wgrad (TN) without materialising transposes.  Operands are 4-D
// TMA tensors (inner, outer, batch_inner, batch_outer) so strided per-head attention operands inside a
// packed qkv buffer are addressed in place.
//
// Capability parity: replaces the XLA-lowered dot ops under timm's Linear layers that the reference
// calls at run_vit_training.py:134-141,153 (qkv / proj / fc1 / fc2 / head) and their autograd
// backward.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <algorithm>
#include <unordered_map>

#include "gemm_sm90.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

namespace {

constexpr int kBlockM = 128;  // rows per CTA: 64 per consumer warpgroup
constexpr int kBlockK = 64;   // 64 bf16 = 128 B = one swizzle atom
constexpr int kMmaK = 16;
constexpr int kConsumerWgs = 2;
constexpr int kNumThreads = 384;  // warpgroup 0: warp0 TMA producer, warp1 AG copier; warpgroups 1-2: wgmma + epilogue
constexpr int kEpiThreads = 128;
constexpr int kCdBufs = 4;            // two 64x64 bf16 staging buffers per consumer warpgroup for TMA stores
constexpr int kCdBufBytes = 64 * 128;  // 64 rows x 128 B

struct KernelParams {
    int M, N, K;
    int batch, nb_inner;
    int m_tiles, n_tiles;  // CTA tiles (128 x BLOCK_N)
    int m_units;           // m-tiles per raster column: m_tiles, or m-tile pairs when CTAs run in 2-CTA clusters
    int n_rot;             // n-tile rotation so that tiles are visited in slab-arrival order (AG fusion)
    int group_n;           // n-tiles per raster group
    GemmEpilogue epi;
    GemmAgFuse ag;
};

constexpr int kAgChunkBytes = 16384;

__device__ __forceinline__ uint4 ld_peer_v4(const void* ptr) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(ptr)
                 : "memory");
    return r;
}
__device__ __forceinline__ void red_release_gpu_add(uint32_t* ptr, uint32_t v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(ptr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* ptr) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ptr) : "memory");
    return v;
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// erf via Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7, far below bf16 resolution): 1 rcp + 1 exp + 6 FMA.
// e = exp(-z^2) is returned too: for z = x/sqrt(2) it is exactly the Gaussian factor gelu'(x) needs.
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float erf_as(float z, float& e) {
    const float az = fabsf(z);
    // rcp.approx (relative error <= 2^-23, below the 1.5e-7 of the formula) rather than __frcp_rn: the correctly
    // rounded reciprocal calls a slow-path subroutine, and the GEMM kernel must stay free of calls (see its body).
    // The argument is >= 1, never in that slow range.
    const float t = rcp_approx(fmaf(0.3275911f, az, 1.0f));
    e = __expf(-az * az);
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float y = 1.0f - poly * t * e;
    return copysignf(y, z);
}
__device__ __forceinline__ float gelu_erf(float x) {
    float e;
    return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f, e));
}
__device__ __forceinline__ float dgelu_erf(float x) {
    float e;
    const float cdf = 0.5f * (1.0f + erf_as(x * 0.70710678118654752f, e));
    return fmaf(x * 0.3989422804014327f, e, cdf);  // cdf + x * pdf,  pdf = exp(-x^2/2)/sqrt(2 pi)
}
// sigmoid(x) = 1 / (1 + exp(-x)) with ex2.approx and rcp.approx: no call.  exp(-x) overflows to inf for x < -88 and the
// reciprocal of inf is 0, so silu(x) = x * sigmoid(x) and silu'(x) = s (1 + x (1 - s)) go to -0 / 0 there, as they should.
__device__ __forceinline__ float sigmoid_approx(float x) { return rcp_approx(1.0f + __expf(-x)); }

// kClusterM = 2: CTAs run in (2, 1, 1) clusters.  The two CTAs of a cluster own m-tiles 2 mp and 2 mp + 1 of the same
// (batch, n-tile), so they need the same B tile: each producer loads its own A tile and one half of B, multicast to
// both CTAs at the same stage offset.  Per k-block a CTA then pulls 16 KB of A + BLOCK_N / 2 rows of B from L2
// instead of 16 KB + BLOCK_N rows.  Stage layout, descriptors and consumer code are the same as with kClusterM = 1;
// only the barrier protocol changes:
//   full_bar[s]  1 arrival (the local producer's expect_tx of the whole stage); the peer's B half completes its bytes
//                here too, possibly before the local expect_tx (the tx count may dip below zero meanwhile).
//   empty_bar[s] 8 * kClusterM arrivals: every consumer warp of BOTH CTAs arrives on both CTAs' barriers, because a
//                producer's multicast writes stage s of the peer as well and may start only once both released it.
// Both CTAs walk the same tile sequence, so they fill and drain the ring in lock step; cluster syncs after barrier
// init and before exit keep a CTA from multicasting into, or arriving on, a peer that has not started or has left.
//
// kGlu (kActSwiglu / kActDSwiglu, 0 otherwise) selects a SwiGLU epilogue (gemm_sm90.h).  A template flag like kRowScale:
// the instantiations with kGlu = 0 compile exactly as they did before the SwiGLU epilogues existed.  The forward GLU
// tile is BLOCK_N / 2 output columns wide: its B stage holds the gate rows [n, n + BLOCK_N / 2) in the lower half and
// the value rows [N + n, ...) in the upper half (with kClusterM = 2, CTA rank 0 loads the gate half and rank 1 the value
// half, at the stage offsets of the plain multicast), so accumulator column j and j + BLOCK_N / 2 pair up in registers.
template <int kMajorA, int kMajorB, int BLOCK_N, int kStages, int kClusterM, bool kRowScale, int kGlu>
__device__ __forceinline__ void gemm_bf16_sm90_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b,
                                                    const CUtensorMap& tmap_d, const CUtensorMap& tmap_aux,
                                                    const KernelParams& p) {
    constexpr int kABytes = kBlockM * kBlockK * 2;
    constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    constexpr int kStageBytes = kABytes + kBBytes;
    constexpr int kTileN = kGlu == kActSwiglu ? BLOCK_N / 2 : BLOCK_N;  // output columns per tile
    static_assert(BLOCK_N % 64 == 0 && BLOCK_N <= 256, "epilogue works in 64-column chunks; wgmma N <= 256");
    static_assert(kABytes % 1024 == 0 && kBBytes % 1024 == 0, "swizzle-128B needs 1024 B aligned stages");
    static_assert(kClusterM == 1 || (kClusterM == 2 && BLOCK_N % 128 == 0), "B splits into two 64-row multiples");
    static_assert(kGlu != kActSwiglu || (kMajorA == 0 && kMajorB == 0 && BLOCK_N % 128 == 0 && !kRowScale),
                  "SwiGLU forward: K-major operands, gate / value halves of 64-row multiples");
    static_assert(kGlu != kActDSwiglu || (kMajorA == 0 && kMajorB == 1 && !kRowScale), "dSwiGLU: the fc2 dgrad (NN)");

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* smem_cd = smem;
    uint8_t* smem_a = smem + kCdBufs * kCdBufBytes;
    uint8_t* smem_b = smem_a + kStages * kABytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_b + kStages * kBBytes);  // [kStages] TMA -> wgmma
    uint64_t* empty_bar = full_bar + kStages;                                       // [kStages] wgmma -> TMA

    const uint32_t warp_idx = threadIdx.x / 32;
    const uint32_t lane = lane_id();
    const uint32_t wg = warp_idx / 4;  // 0: producer + all-gather copier, 1-2: consumers
    // No printf anywhere in this kernel: a printf is a function call, and any call in a kernel that uses wgmma makes
    // ptxas serialise every wgmma (warning C7510: each MMA then waits for the previous one).  Faults trap silently.
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();  // SWIZZLE_128B tiles need 1024-B alignment

    if (warp_idx == 0 && elect_one()) {
        prefetch_tmap(&tmap_a);
        prefetch_tmap(&tmap_b);
        prefetch_tmap(&tmap_d);
        if (p.epi.has_aux_out) prefetch_tmap(&tmap_aux);
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&full_bar[i], 1);                              // the producer's expect_tx arrive
            mbar_init(&empty_bar[i], kConsumerWgs * 4 * kClusterM);  // lane 0 of every consumer warp of the cluster
        }
        fence_mbar_init();
    }
    if constexpr (kClusterM > 1)
        cluster_sync();  // the peer's barriers are initialised before anything is multicast to or arrives on them
    else
        __syncthreads();

    // A unit is one tile (kClusterM = 1) or one cluster's pair of vertically adjacent tiles (kClusterM = 2).
    // The rank is re-read from its special register where used: the consumers run at the register limit.
    auto cta_rank = [] { return kClusterM > 1 ? static_cast<int>(cluster_ctarank()) : 0; };
    const int units_per_batch = p.m_units * p.n_tiles;
    const int total_units = units_per_batch * p.batch;
    const int num_kb = (p.K + kBlockK - 1) / kBlockK;
    const int kGroupN = p.group_n;  // n-tiles per raster group (keeps a wave's A/B footprint L2-resident)

    // Static persistent schedule: CTA (or cluster) c computes units c, c + grid, c + 2 grid, ...  The units in flight
    // are a contiguous window of the raster, so co-running CTAs share A / B panels in L2.
    // With an odd m-tile count the second CTA of the last pair gets m-tile m_tiles, wholly below the matrix.  It still
    // runs the full protocol (its B half feeds the peer, its consumers release the peer's stages).  Its A box is
    // wholly out of bounds: TMA fills it with zeros and still counts its bytes (the kernel relies on that already for
    // the out-of-range 64-row boxes of MN-major operands), and its output rows are clipped by the TMA store and zeroed
    // for the column sums like any row >= M.  Keeping the load avoids a second producer path for one tile per column.
    auto decode_tile = [&](int t, int& b, int& mt, int& nt) {
        b = t / units_per_batch;
        const int r = t - b * units_per_batch;
        const int per_group = p.m_units * kGroupN;
        const int g = r / per_group;
        const int first_n = g * kGroupN;
        const int gsz = min(kGroupN, p.n_tiles - first_n);
        const int in_g = r - g * per_group;
        mt = (in_g / gsz) * kClusterM + cta_rank();
        nt = first_n + in_g % gsz;
        nt += p.n_rot;  // AG fusion: start with the n-tiles of the locally owned slab
        if (nt >= p.n_tiles) nt -= p.n_tiles;
    };
    const int ag_chunks_per_slab =
        p.ag.world > 1 ? static_cast<int>((p.ag.slab_bytes + kAgChunkBytes - 1) / kAgChunkBytes) : 0;

    if (wg == 0) {
        reg_dealloc<56>();
        if (warp_idx == 0) {
            // ================================= TMA producer =================================
            if (elect_one()) {
                uint32_t stage = 0, phase = 0;
                for (int t = blockIdx.x / kClusterM; t < total_units; t += gridDim.x / kClusterM) {
                    int b, mt, nt;
                    decode_tile(t, b, mt, nt);
                    const int bi = b % p.nb_inner, bo = b / p.nb_inner;
                    const int m_idx = mt * kBlockM;
                    const int n_idx = nt * kTileN;
                    if (p.ag.world > 1) {
                        // B rows [n_idx, n_idx + BLOCK_N) must have been pulled into the local gathered buffer
                        const int last_row = min(n_idx + BLOCK_N, p.N) - 1;
                        if (last_row >= n_idx) {
                            const int s_lo = min(n_idx / p.ag.rows_per_slab, p.ag.world - 1);
                            const int s_hi = min(last_row / p.ag.rows_per_slab, p.ag.world - 1);
                            for (int sl = s_lo; sl <= s_hi; ++sl) {
                                uint32_t spins = 0;
                                while (ld_acquire_gpu(p.ag.flags + sl) < static_cast<uint32_t>(ag_chunks_per_slab)) {
                                    if (++spins > (1u << 26)) __trap();  // slab never arrived
                                }
                            }
                            fence_proxy_async_all();  // generic-proxy peer copies -> async-proxy (TMA) reads
                        }
                    }
                    for (int kb = 0; kb < num_kb; ++kb) {
                        mbar_wait_silent(&empty_bar[stage], phase ^ 1);
                        const int k_idx = kb * kBlockK;
                        uint8_t* sa = smem_a + stage * kABytes;
                        uint8_t* sb = smem_b + stage * kBBytes;
                        mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);  // out-of-bounds box parts count too
                        if constexpr (kMajorA == 0) {
                            tma_load_4d(&tmap_a, &full_bar[stage], sa, k_idx, m_idx, bi, bo);
                        } else {
#pragma unroll
                            for (int i = 0; i < kBlockM / 64; ++i)
                                tma_load_4d(&tmap_a, &full_bar[stage], sa + i * (64 * kBlockK * 2), m_idx + i * 64,
                                                 k_idx, bi, bo);
                        }
                        if constexpr (kGlu == kActSwiglu) {
                            // gate rows [n_idx, +BLOCK_N / 2) -> lower half, value rows [N + n_idx, ...) -> upper half.
                            // Gate rows past N are value rows (their columns are discarded), value rows past 2N are
                            // zero-filled by TMA, so any N works.
                            constexpr int kHalfN = BLOCK_N / 2;
                            if constexpr (kClusterM == 1) {
                                tma_load_4d(&tmap_b, &full_bar[stage], sb, k_idx, n_idx, bi, bo);
                                tma_load_4d(&tmap_b, &full_bar[stage], sb + kHalfN * (kBlockK * 2), k_idx, p.N + n_idx,
                                            bi, bo);
                            } else {
                                const int r = cta_rank();
                                tma_load_4d_multicast(&tmap_b, &full_bar[stage], sb + r * kHalfN * (kBlockK * 2), k_idx,
                                                      n_idx + r * p.N, bi, bo, 0b11);
                            }
                        } else if constexpr (kClusterM == 1) {
                            if constexpr (kMajorB == 0) {
                                tma_load_4d(&tmap_b, &full_bar[stage], sb, k_idx, n_idx, bi, bo);
                            } else {
#pragma unroll
                                for (int i = 0; i < BLOCK_N / 64; ++i)
                                    tma_load_4d(&tmap_b, &full_bar[stage], sb + i * (64 * kBlockK * 2), n_idx + i * 64,
                                                k_idx, bi, bo);
                            }
                        } else {
                            // this CTA's half of B: rows [n_idx + h, n_idx + h + BLOCK_N / 2), h = rank * BLOCK_N / 2,
                            // to stage offset h * 128 B in both CTAs (the (64, BLOCK_N / 2) box of a K-major B is
                            // laid out exactly like the lower or upper half of the (64, BLOCK_N) box)
                            constexpr int kHalfN = BLOCK_N / 2;
                            const int h = cta_rank() * kHalfN;
                            if constexpr (kMajorB == 0) {
                                tma_load_4d_multicast(&tmap_b, &full_bar[stage], sb + h * (kBlockK * 2), k_idx,
                                                      n_idx + h, bi, bo, 0b11);
                            } else {
#pragma unroll
                                for (int i = 0; i < kHalfN / 64; ++i)
                                    tma_load_4d_multicast(&tmap_b, &full_bar[stage],
                                                          sb + (h / 64 + i) * (64 * kBlockK * 2), n_idx + h + i * 64,
                                                          k_idx, bi, bo, 0b11);
                            }
                        }
                        stage = (stage + 1 == kStages) ? 0 : stage + 1;
                        phase ^= (stage == 0);
                    }
                }
            }
        } else if (warp_idx == 1) {
            // ================================= All-gather copier (AG fusion only) =================================
            if (p.ag.world > 1) {
                const int total_chunks = p.ag.world * ag_chunks_per_slab;
                uint32_t* chunk_counter = p.ag.flags + p.ag.world;  // zeroed with the flags
                for (;;) {
                    int c = 0;
                    if (lane == 0) c = static_cast<int>(atomicAdd(chunk_counter, 1u));
                    c = __shfl_sync(0xffffffffu, c, 0);
                    if (c >= total_chunks) break;
                    const int k = c / ag_chunks_per_slab;            // arrival index: 0 = own slab
                    const int sl = (p.ag.rank + k) % p.ag.world;      // slab pulled now (ranks start at different peers)
                    const int64_t off = static_cast<int64_t>(c - k * ag_chunks_per_slab) * kAgChunkBytes;
                    const int64_t nbytes = min(static_cast<int64_t>(kAgChunkBytes), p.ag.slab_bytes - off);
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.ag.peer_src[sl]) + off;
                    uint8_t* dst = static_cast<uint8_t*>(p.ag.dst) + static_cast<int64_t>(sl) * p.ag.slab_bytes + off;
                    const int nvec = static_cast<int>(nbytes / 16);
                    int i = lane;
                    for (; i + 3 * 32 < nvec; i += 4 * 32) {
                        uint4 v[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) v[u] = ld_peer_v4(src + static_cast<int64_t>(i + u * 32) * 16);
#pragma unroll
                        for (int u = 0; u < 4; ++u) *reinterpret_cast<uint4*>(dst + static_cast<int64_t>(i + u * 32) * 16) = v[u];
                    }
                    for (; i < nvec; i += 32) *reinterpret_cast<uint4*>(dst + static_cast<int64_t>(i) * 16) = ld_peer_v4(src + static_cast<int64_t>(i) * 16);
                    __threadfence();
                    __syncwarp();
                    if (lane == 0) red_release_gpu_add(p.ag.flags + sl, 1);
                }
            }
        }
    } else {
        // ================================= Consumer warpgroups: wgmma + epilogue =================================
        // Warpgroup w owns rows [64 w, 64 w + 64) of the 128 x BLOCK_N tile: one m64nNk16 wgmma per 16-wide k step,
        // fp32 accumulators in registers.  One k-block of MMAs stays in flight while the next one is issued; the smem
        // slot of a k-block is handed back to the producer as soon as its MMAs retired.
        reg_alloc<224>();
        const uint32_t cw = wg - 1;                       // consumer warpgroup index = 64-row slab of the tile
        const uint32_t etid = threadIdx.x & 127;
        const uint32_t wrow = (warp_idx & 3) * 16 + lane / 4;  // this thread's accumulator rows: wrow and wrow + 8
        const uint32_t cpair = (lane & 3) * 2;            // first of its two adjacent columns inside every 8-column group
        const uint32_t bar_id = 1 + cw;
        uint8_t* const grp_buf = smem_cd + cw * 2 * kCdBufBytes;  // two 64 x 64 staging buffers per warpgroup
        const GemmEpilogue& e = p.epi;
        const bool ext_is_aux = e.act == kActDGelu;
        // K-major : 8-row groups are 1024 B apart (SBO); one swizzle atom along K so LBO is unused.
        // MN-major: 8-k groups are 1024 B apart (SBO); 64-wide MN atoms are BLOCK_K * 128 B apart (LBO).
        constexpr uint32_t kLbo = kBlockK * 128;
        constexpr uint32_t kKStepA = kMajorA == 0 ? (kMmaK * 2) : (kMmaK * 128);  // bytes per 16-wide k step
        constexpr uint32_t kKStepB = kMajorB == 0 ? (kMmaK * 2) : (kMmaK * 128);
        constexpr uint32_t kSlabA = 64 * kBlockK * 2;     // both majors: the warpgroup's 64 rows are 8 KB further
        uint32_t stage = 0, phase = 0;
        uint32_t flip = 0;
        float d[BLOCK_N / 2];
        // hand stage s back to the producers that write it: this CTA's, and with multicast the peer's too
        auto release = [&](uint32_t s) {
            if constexpr (kClusterM == 1) {
                mbar_arrive(&empty_bar[s]);
            } else {
#pragma unroll
                for (int c = 0; c < kClusterM; ++c) mbar_arrive_cluster(&empty_bar[s], c);
            }
        };

        for (int t = blockIdx.x / kClusterM; t < total_units; t += gridDim.x / kClusterM) {
            int b, mt, nt;
            decode_tile(t, b, mt, nt);
            const int bi = b % p.nb_inner, bo = b / p.nb_inner;
            const int m0 = mt * kBlockM + cw * 64;
            const int n0 = nt * kTileN;

            uint32_t prev_stage = 0;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait_silent(&full_bar[stage], phase);
                const uint32_t a_addr = smem_u32(smem_a + stage * kABytes) + cw * kSlabA;
                const uint32_t b_addr = smem_u32(smem_b + stage * kBBytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / kMmaK; ++k) {
                    const uint64_t da = make_wgmma_desc(a_addr + k * kKStepA, kLbo, 1024, 1);
                    const uint64_t db = make_wgmma_desc(b_addr + k * kKStepB, kLbo, 1024, 1);
                    WgmmaSS<BLOCK_N, kMajorA, kMajorB>::mma(d, da, db, (kb > 0 || k > 0) ? 1u : 0u);
                }
                wgmma_commit();
                if (kb > 0) {
                    wgmma_wait<1>();  // the previous k-block's MMAs are done reading their slot
                    if (lane == 0) release(prev_stage);
                }
                prev_stage = stage;
                stage = (stage + 1 == kStages) ? 0 : stage + 1;
                phase ^= (stage == 0);
            }
            wgmma_wait<0>();
            if (lane == 0) release(prev_stage);

            // ---- epilogue: registers -> swizzled staging buffer -> TMA store, 64 columns at a time ----
            const int row0 = m0 + static_cast<int>(wrow), row1 = row0 + 8;
            const bool row0_ok = row0 < p.M, row1_ok = row1 < p.M;
            if constexpr (kGlu == kActSwiglu) {
                // gate of output column n in accumulator chunk c, its value in chunk c + kHalfChunks
                constexpr int kHalfChunks = BLOCK_N / 128;
                auto gate_value = [&](int c, int j, float (&a)[4], float (&v)[4]) {
#pragma unroll
                    for (int q = 0; q < 4; ++q) a[q] = d[(c * 8 + j) * 4 + q], v[q] = d[((c + kHalfChunks) * 8 + j) * 4 + q];
                };
#pragma unroll
                for (int c = 0; c < kHalfChunks; ++c) {
                    const int ncol0 = n0 + c * 64;
                    if (ncol0 >= p.N) continue;  // warpgroup-uniform
                    // both biases go into the accumulators in place: no bias value stays live across the two passes
                    if (e.bias != nullptr) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int col = ncol0 + j * 8 + static_cast<int>(cpair);
                            if (col < p.N) {
                                const uint32_t bg = __ldg(reinterpret_cast<const uint32_t*>(e.bias + col));
                                const uint32_t bv = __ldg(reinterpret_cast<const uint32_t*>(e.bias + p.N + col));
                                float* dg = d + (c * 8 + j) * 4;
                                float* dv = d + ((c + kHalfChunks) * 8 + j) * 4;
                                dg[0] += bf16_lo(bg), dg[1] += bf16_hi(bg), dg[2] += bf16_lo(bg), dg[3] += bf16_hi(bg);
                                dv[0] += bf16_lo(bv), dv[1] += bf16_hi(bv), dv[2] += bf16_lo(bv), dv[3] += bf16_hi(bv);
                            }
                        }
                    }
                    // Three outputs per chunk and two staging buffers: the pre-activations go first (gate -> buffer 0,
                    // value -> buffer 1, stored to the two [M, N] halves of u through the aux map's batch index), then
                    // g reuses buffer 0 once the TMA engine has read it.  Without them g alternates between buffers.
                    if (e.has_aux_out) {
                        if (etid == 0) tma_store_wait_read<0>();
                        named_bar_sync(bar_id, kEpiThreads);
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            float a[4], v[4];
                            gate_value(c, j, a, v);
                            const uint32_t off0 = wrow * 128 + ((j ^ (wrow & 7)) * 16) + cpair * 2;
                            st_shared_b32(smem_u32(grp_buf) + off0, pack_bf16x2(a[0], a[1]));
                            st_shared_b32(smem_u32(grp_buf) + off0 + 8 * 128, pack_bf16x2(a[2], a[3]));
                            st_shared_b32(smem_u32(grp_buf + kCdBufBytes) + off0, pack_bf16x2(v[0], v[1]));
                            st_shared_b32(smem_u32(grp_buf + kCdBufBytes) + off0 + 8 * 128, pack_bf16x2(v[2], v[3]));
                        }
                        fence_proxy_async_smem();
                        named_bar_sync(bar_id, kEpiThreads);
                        if (etid == 0) {
                            tma_store_4d(&tmap_aux, grp_buf, ncol0, m0, 0, 0);
                            tma_store_4d(&tmap_aux, grp_buf + kCdBufBytes, ncol0, m0, 1, 0);
                            tma_store_commit();
                            tma_store_wait_read<0>();
                        }
                    } else if (etid == 0) {
                        tma_store_wait_read<1>();
                    }
                    named_bar_sync(bar_id, kEpiThreads);
                    uint8_t* buf0 = grp_buf + (e.has_aux_out ? 0 : (flip & 1)) * kCdBufBytes;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        float a[4], v[4];
                        gate_value(c, j, a, v);
#pragma unroll
                        for (int q = 0; q < 4; ++q) v[q] *= a[q] * sigmoid_approx(a[q]);
                        const uint32_t off0 = wrow * 128 + ((j ^ (wrow & 7)) * 16) + cpair * 2;
                        st_shared_b32(smem_u32(buf0) + off0, pack_bf16x2(v[0], v[1]));
                        st_shared_b32(smem_u32(buf0) + off0 + 8 * 128, pack_bf16x2(v[2], v[3]));
                    }
                    fence_proxy_async_smem();
                    named_bar_sync(bar_id, kEpiThreads);
                    if (etid == 0) {
                        tma_store_4d(&tmap_d, buf0, ncol0, m0, bi, bo);
                        tma_store_commit();
                    }
                    ++flip;
                }
            } else if constexpr (kGlu == kActDSwiglu) {
                // acc = dh[m, n]; a = u[m, n] (gate), b = u[m, N + n] (value).  du_gate -> buffer 0 -> D map,
                // du_val -> buffer 1 -> aux map (the two-buffer staging of the pre-activation side output).
                const __nv_bfloat16* u0 = e.aux_in + static_cast<int64_t>(row0) * e.ld_aux;
                const __nv_bfloat16* u1 = e.aux_in + static_cast<int64_t>(row1) * e.ld_aux;
#pragma unroll
                for (int c = 0; c < BLOCK_N / 64; ++c) {
                    const int ncol0 = n0 + c * 64;
                    if (ncol0 >= p.N) continue;  // warpgroup-uniform
                    uint8_t* buf0 = grp_buf;
                    uint8_t* buf1 = grp_buf + kCdBufBytes;
                    if (etid == 0) tma_store_wait_read<0>();
                    named_bar_sync(bar_id, kEpiThreads);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int col = ncol0 + j * 8 + static_cast<int>(cpair);
                        const bool c_ok = col < p.N;  // N % 8 == 0: col and col + 1 together
                        uint32_t xa[2] = {0, 0}, xb[2] = {0, 0};
                        if (c_ok) {
                            if (row0_ok) {
                                xa[0] = __ldg(reinterpret_cast<const uint32_t*>(u0 + col));
                                xb[0] = __ldg(reinterpret_cast<const uint32_t*>(u0 + p.N + col));
                            }
                            if (row1_ok) {
                                xa[1] = __ldg(reinterpret_cast<const uint32_t*>(u1 + col));
                                xb[1] = __ldg(reinterpret_cast<const uint32_t*>(u1 + p.N + col));
                            }
                        }
                        float dg[4], dv[4];
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const float a = (q & 1) ? bf16_hi(xa[q >> 1]) : bf16_lo(xa[q >> 1]);
                            const float b = (q & 1) ? bf16_hi(xb[q >> 1]) : bf16_lo(xb[q >> 1]);
                            const float dh = d[(c * 8 + j) * 4 + q];
                            const float sg = sigmoid_approx(a);
                            const bool ok = c_ok && ((q >> 1) ? row1_ok : row0_ok);
                            dv[q] = ok ? dh * (a * sg) : 0.f;  // zeros keep the column sums clean
                            dg[q] = ok ? dh * b * (sg * fmaf(a, 1.0f - sg, 1.0f)) : 0.f;
                        }
                        const uint32_t off0 = wrow * 128 + ((j ^ (wrow & 7)) * 16) + cpair * 2;
                        st_shared_b32(smem_u32(buf0) + off0, pack_bf16x2(dg[0], dg[1]));
                        st_shared_b32(smem_u32(buf0) + off0 + 8 * 128, pack_bf16x2(dg[2], dg[3]));
                        st_shared_b32(smem_u32(buf1) + off0, pack_bf16x2(dv[0], dv[1]));
                        st_shared_b32(smem_u32(buf1) + off0 + 8 * 128, pack_bf16x2(dv[2], dv[3]));
                    }
                    fence_proxy_async_smem();
                    named_bar_sync(bar_id, kEpiThreads);
                    if (etid == 0) {
                        tma_store_4d(&tmap_d, buf0, ncol0, m0, bi, bo);
                        tma_store_4d(&tmap_aux, buf1, ncol0, m0, bi, bo);
                        tma_store_commit();
                    }
                    if (e.colsum != nullptr) {
                        // fc1 bias gradient: column n of du_gate -> colsum[n], of du_val -> colsum[N + n]
                        const int ccol = etid & 63;
                        const int rhalf = etid >> 6;
                        const int jj = ccol >> 3, within = ccol & 7;
                        float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
                        for (int r = 0; r < 32; ++r) {
                            const int rr = rhalf * 32 + r;
                            const int off = rr * 128 + ((jj ^ (rr & 7)) * 16) + within * 2;
                            s0 += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(buf0 + off));
                            s1 += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(buf1 + off));
                        }
                        if (ncol0 + ccol < p.N) {
                            atomicAdd(e.colsum + ncol0 + ccol, s0);
                            atomicAdd(e.colsum + p.N + ncol0 + ccol, s1);
                        }
                    }
                    ++flip;
                }
            } else {
                const __nv_bfloat16 *ext0 = nullptr, *ext1 = nullptr;
                if (ext_is_aux) {
                    ext0 = e.aux_in + static_cast<int64_t>(row0) * e.ld_aux;
                    ext1 = e.aux_in + static_cast<int64_t>(row1) * e.ld_aux;
                } else if (e.residual != nullptr) {
                    ext0 = e.residual + static_cast<int64_t>(e.res_row_mod > 0 ? row0 % e.res_row_mod : row0) * e.ld_res;
                    ext1 = e.residual + static_cast<int64_t>(e.res_row_mod > 0 ? row1 % e.res_row_mod : row1) * e.ld_res;
                }
                // kRowScale (stochastic depth): v = (acc + bias) * row_scale[row / rows_per_scale] before the residual add,
                // the scale read once per accumulator row of the tile.  A template flag rather than a run-time branch: the
                // GELU / dGELU epilogues run at the register limit, and any change to their code changes how ptxas
                // schedules them; the instantiations without the flag compile exactly as they would without the feature.
                float rs0 = 1.f, rs1 = 1.f;
                if constexpr (kRowScale) {
                    if (row0_ok) rs0 = __ldg(e.row_scale + row0 / e.rows_per_scale);
                    if (row1_ok) rs1 = __ldg(e.row_scale + row1 / e.rows_per_scale);
                }
    #pragma unroll
                for (int c = 0; c < BLOCK_N / 64; ++c) {
                    const int ncol0 = n0 + c * 64;
                    if (ncol0 >= p.N) continue;  // warpgroup-uniform: nothing to store
                    uint8_t* buf0 = grp_buf + (e.has_aux_out ? 0 : (flip & 1)) * kCdBufBytes;
                    uint8_t* buf1 = grp_buf + kCdBufBytes;
                    if (etid == 0) {  // staging buffer(s) of this warpgroup free again?
                        if (e.has_aux_out)
                            tma_store_wait_read<0>();
                        else
                            tma_store_wait_read<1>();
                    }
                    named_bar_sync(bar_id, kEpiThreads);
    #pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int col = ncol0 + j * 8 + static_cast<int>(cpair);
                        const bool c0_ok = col < p.N, c1_ok = col + 1 < p.N;
                        float v[4] = {d[(c * 8 + j) * 4], d[(c * 8 + j) * 4 + 1], d[(c * 8 + j) * 4 + 2], d[(c * 8 + j) * 4 + 3]};
                        uint32_t x0 = 0, x1 = 0;  // dGELU pre-activation or residual of (row0 | row1, col..col+1)
                        if (ext0 != nullptr && c0_ok) {
                            if (row0_ok) x0 = __ldg(reinterpret_cast<const uint32_t*>(ext0 + col));
                            if (row1_ok) x1 = __ldg(reinterpret_cast<const uint32_t*>(ext1 + col));
                        }
                        if (e.bias != nullptr && c0_ok) {
                            const uint32_t bw = __ldg(reinterpret_cast<const uint32_t*>(e.bias + col));
                            v[0] += bf16_lo(bw), v[1] += bf16_hi(bw), v[2] += bf16_lo(bw), v[3] += bf16_hi(bw);
                        }
                        // 16-byte chunk j of a 128-byte row, XOR-swizzled with the row like the TMA store expects
                        const uint32_t off0 = wrow * 128 + ((j ^ (wrow & 7)) * 16) + cpair * 2;
                        const uint32_t off1 = off0 + 8 * 128;  // row + 8 has the same (row & 7)
                        if (e.has_aux_out) {
                            st_shared_b32(smem_u32(buf1) + off0, pack_bf16x2(v[0], v[1]));
                            st_shared_b32(smem_u32(buf1) + off1, pack_bf16x2(v[2], v[3]));
                        }
                        if (e.act == kActGelu) {
    #pragma unroll
                            for (int q = 0; q < 4; ++q) v[q] = gelu_erf(v[q]);
                        } else if (ext_is_aux) {
                            v[0] *= dgelu_erf(bf16_lo(x0)), v[1] *= dgelu_erf(bf16_hi(x0));
                            v[2] *= dgelu_erf(bf16_lo(x1)), v[3] *= dgelu_erf(bf16_hi(x1));
                        }
                        if constexpr (kRowScale) {  // host: only with kActNone, so this is (acc + bias) * scale
                            v[0] *= rs0, v[1] *= rs0, v[2] *= rs1, v[3] *= rs1;
                        }
                        if (e.residual != nullptr && !ext_is_aux) {
                            v[0] += bf16_lo(x0), v[1] += bf16_hi(x0), v[2] += bf16_lo(x1), v[3] += bf16_hi(x1);
                        }
                        // rows / columns outside the problem are clipped by the TMA store; zeros keep the column sums clean
                        if (!(row0_ok && c0_ok)) v[0] = 0.f;
                        if (!(row0_ok && c1_ok)) v[1] = 0.f;
                        if (!(row1_ok && c0_ok)) v[2] = 0.f;
                        if (!(row1_ok && c1_ok)) v[3] = 0.f;
                        st_shared_b32(smem_u32(buf0) + off0, pack_bf16x2(v[0], v[1]));
                        st_shared_b32(smem_u32(buf0) + off1, pack_bf16x2(v[2], v[3]));
                    }
                    fence_proxy_async_smem();
                    named_bar_sync(bar_id, kEpiThreads);
                    if (etid == 0) {
                        tma_store_4d(&tmap_d, buf0, ncol0, m0, bi, bo);
                        tma_store_commit();
                        if (e.has_aux_out) {
                            tma_store_4d(&tmap_aux, buf1, ncol0, m0, bi, bo);
                            tma_store_commit();
                        }
                    }
                    if (e.colsum != nullptr) {
                        // Bias gradient: column sums of the (bf16-rounded) output tile, fp32 atomics.
                        const int ccol = etid & 63;       // column within the chunk
                        const int rhalf = etid >> 6;      // 0/1 -> rows [0,32) / [32,64)
                        const int jj = ccol >> 3, within = ccol & 7;
                        float s = 0.f;
    #pragma unroll 8
                        for (int r = 0; r < 32; ++r) {
                            const int rr = rhalf * 32 + r;
                            const uint8_t* ptr = buf0 + rr * 128 + ((jj ^ (rr & 7)) * 16) + within * 2;
                            s += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(ptr));
                        }
                        if (ncol0 + ccol < p.N)
                            atomicAdd(e.colsum + static_cast<int64_t>(bi) * e.colsum_bi_stride + ncol0 + ccol, s);
                    }
                    ++flip;
                }
            }
        }
        if (etid == 0) tma_store_wait<0>();
    }
    if constexpr (kClusterM > 1) {
        // the peer's last multicasts into this CTA have landed (our consumers waited for them), but its consumers may
        // still be about to arrive on our empty barriers: leave only together
        __syncwarp();
        cluster_sync();
    }
}

template <int kMajorA, int kMajorB, int BLOCK_N, int kStages, int kClusterM, bool kRowScale>
__global__ void __launch_bounds__(kNumThreads, 1)
    gemm_bf16_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                          const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_aux,
                          const KernelParams p) {
    gemm_bf16_sm90_body<kMajorA, kMajorB, BLOCK_N, kStages, kClusterM, kRowScale, 0>(tmap_a, tmap_b, tmap_d, tmap_aux, p);
}

// SwiGLU forward (kGlu = kActSwiglu, K-major B) and fc2 dgrad (kActDSwiglu, MN-major B); A is K-major in both.
template <int kMajorB, int BLOCK_N, int kStages, int kClusterM, int kGlu>
__global__ void __launch_bounds__(kNumThreads, 1)
    gemm_glu_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                         const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_aux,
                         const KernelParams p) {
    gemm_bf16_sm90_body<0, kMajorB, BLOCK_N, kStages, kClusterM, false, kGlu>(tmap_a, tmap_b, tmap_d, tmap_aux, p);
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode_fn() {
    static EncodeFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres);
        if (err != cudaSuccess || qres != cudaDriverEntryPointSuccess || sym == nullptr)
            throw std::runtime_error("cuTensorMapEncodeTiled not available from the driver");
        fn = reinterpret_cast<EncodeFn>(sym);
    });
    return fn;
}

struct TmapKey {
    uint64_t ptr;
    int64_t d[4];
    int64_t s[3];
    int32_t box[2];
    bool operator==(const TmapKey& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
        size_t h = 1469598103934665603ull;
        for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
        return h;
    }
};

// 4-D bf16 tensor map: dims (inner, outer, batch_inner, batch_outer), box (box_inner, box_outer, 1, 1).
CUtensorMap make_tmap(const GemmOperand& op, int64_t inner, int64_t outer, int box_inner, int box_outer,
                      int swizzle_bytes = 128) {
    static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
    static std::mutex mu;
    TmapKey key;
    std::memset(&key, 0, sizeof(key));
    key.ptr = reinterpret_cast<uint64_t>(op.ptr);
    key.d[0] = inner, key.d[1] = outer, key.d[2] = op.nb_inner, key.d[3] = op.nb_outer;
    key.s[0] = op.ld, key.s[1] = op.stride_b_inner, key.s[2] = op.stride_b_outer;
    key.box[0] = box_inner, key.box[1] = box_outer + (swizzle_bytes << 16);
    {
        std::lock_guard<std::mutex> lock(mu);
        auto it = cache.find(key);
        if (it != cache.end()) return it->second;
    }
    if ((reinterpret_cast<uint64_t>(op.ptr) & 15) != 0) throw std::runtime_error("gemm: operand base must be 16 B aligned");
    if ((op.ld * 2) % 16 != 0) throw std::runtime_error("gemm: leading dimension must be a multiple of 8 elements");
    CUtensorMap tm;
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(outer),
                          static_cast<cuuint64_t>(op.nb_inner), static_cast<cuuint64_t>(op.nb_outer)};
    // Strides of size-1 batch dims are irrelevant but must still be legal multiples of 16 B.
    const int64_t sbi = op.nb_inner > 1 ? op.stride_b_inner : op.ld * outer;
    const int64_t sbo = op.nb_outer > 1 ? op.stride_b_outer : sbi * op.nb_inner;
    if ((sbi * 2) % 16 != 0 || (sbo * 2) % 16 != 0) throw std::runtime_error("gemm: batch strides must be multiples of 8 elements");
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(op.ld * 2), static_cast<cuuint64_t>(sbi * 2),
                             static_cast<cuuint64_t>(sbo * 2)};
    cuuint32_t box[4] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_outer), 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult res = get_encode_fn()(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(op.ptr), dims, strides,
                                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                   : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                         : CU_TENSOR_MAP_SWIZZLE_32B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (res != CUDA_SUCCESS) {
        char msg[256];
        snprintf(msg, sizeof(msg),
                 "cuTensorMapEncodeTiled failed (%d): dims=(%lld,%lld,%lld,%lld) ld=%lld box=(%d,%d)", (int)res,
                 (long long)inner, (long long)outer, (long long)op.nb_inner, (long long)op.nb_outer, (long long)op.ld,
                 box_inner, box_outer);
        throw std::runtime_error(msg);
    }
    std::lock_guard<std::mutex> lock(mu);
    if (cache.size() > 4096) cache.clear();
    cache.emplace(key, tm);
    return tm;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}

void check(cudaError_t err, const char* what) {
    if (err != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(err));
}

template <int kMajorA, int kMajorB, int BLOCK_N, int kStages, int kClusterM, bool kRowScale, int kGlu>
constexpr auto kernel_for() {
    if constexpr (kGlu == 0)
        return gemm_bf16_sm90_kernel<kMajorA, kMajorB, BLOCK_N, kStages, kClusterM, kRowScale>;
    else
        return gemm_glu_sm90_kernel<kMajorB, BLOCK_N, kStages, kClusterM, kGlu>;
}

template <int kMajorA, int kMajorB, int BLOCK_N, int kStages, int kClusterM, bool kRowScale = false, int kGlu = 0>
void launch(const GemmOperand& A, const GemmOperand& B, const GemmOperand& D, const GemmOperand* aux, int M, int N,
            int K, const GemmEpilogue& epi, int max_ctas, cudaStream_t stream, const GemmAgFuse* ag) {
    constexpr int kSmem = kCdBufs * kCdBufBytes + kStages * (kBlockM + BLOCK_N) * kBlockK * 2 + 2 * kStages * 8;
    static_assert(kSmem <= 232448, "shared memory budget exceeded (227 KB per block on sm_90)");
    constexpr int kTileN = kGlu == kActSwiglu ? BLOCK_N / 2 : BLOCK_N;
    auto kern = kernel_for<kMajorA, kMajorB, BLOCK_N, kStages, kClusterM, kRowScale, kGlu>();
    static bool attr_set = false;
    if (!attr_set) {
        check(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem), "cudaFuncSetAttribute");
        attr_set = true;
    }
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute cluster_attr;
    cluster_attr.id = cudaLaunchAttributeClusterDimension;
    cluster_attr.val.clusterDim.x = kClusterM, cluster_attr.val.clusterDim.y = 1, cluster_attr.val.clusterDim.z = 1;
    cfg.blockDim = dim3(kNumThreads);
    cfg.dynamicSmemBytes = kSmem;
    cfg.stream = stream;
    cfg.attrs = &cluster_attr;
    cfg.numAttrs = kClusterM > 1 ? 1 : 0;
    // Clusters that can be resident at once: a cluster's CTAs must share a GPC, so with one CTA per SM this can be
    // fewer than num_sms / 2.  The schedule is a static stride over a persistent grid, so one cluster more than fits
    // would run as a second wave after the first and about double the GEMM's time.
    static int resident_units = 0;
    if (resident_units == 0) {
        if constexpr (kClusterM == 1) {
            resident_units = num_sms();
        } else {
            cfg.gridDim = dim3(num_sms() / kClusterM * kClusterM);
            check(cudaOccupancyMaxActiveClusters(&resident_units, kern, &cfg), "cudaOccupancyMaxActiveClusters");
            if (resident_units < 1) throw std::runtime_error("gemm: no 2-CTA cluster of this kernel fits an SM pair");
        }
    }
    // A: K-major -> (inner=K, outer=M), box (64, 128).  MN-major -> (inner=M, outer=K), box (64, 64).
    // B: K-major -> box (64, BLOCK_N / kClusterM): each CTA of a cluster loads its share.  MN-major -> box (64, 64).
    CUtensorMap ta = kMajorA == 0 ? make_tmap(A, K, M, kBlockK, kBlockM) : make_tmap(A, M, K, 64, kBlockK);
    // SwiGLU forward: B is the whole [2N, K] weight, read in (64, BLOCK_N / 2) gate and value boxes, and the aux output
    // u [M, 2N] is viewed as two [M, N] halves (batch index 0 = gate, 1 = value; the second starts at column N, which
    // is why N must be a multiple of 8).
    CUtensorMap tb = kGlu == kActSwiglu ? make_tmap(B, K, 2 * static_cast<int64_t>(N), kBlockK, BLOCK_N / 2)
                     : kMajorB == 0     ? make_tmap(B, K, N, kBlockK, BLOCK_N / kClusterM)
                                        : make_tmap(B, N, K, 64, kBlockK);
    CUtensorMap td = make_tmap(D, N, M, 64, 64);
    CUtensorMap tx = td;
    if (epi.has_aux_out && aux != nullptr) {
        GemmOperand x = *aux;
        if (kGlu == kActSwiglu) x.nb_inner = 2, x.stride_b_inner = N;
        tx = make_tmap(x, N, M, 64, 64);
    }

    KernelParams p;
    p.M = M, p.N = N, p.K = K;
    p.batch = static_cast<int>(D.nb_inner * D.nb_outer);
    p.nb_inner = static_cast<int>(D.nb_inner);
    p.m_tiles = (M + kBlockM - 1) / kBlockM;
    p.m_units = (p.m_tiles + kClusterM - 1) / kClusterM;
    p.n_tiles = (N + kTileN - 1) / kTileN;
    p.epi = epi;
    p.n_rot = 0;
    // n-tiles per raster group: 2048 output columns.  Reasoning, not a measurement: a wave of 132 CTAs then covers
    // ~16 m-tiles x 2048 columns, about as many A rows (2112) as B rows (2048), the split that fetches the fewest
    // operand bytes per wave, and at K = 5120 both panels together (~43 MB) are below the 50 MB of L2.
    p.group_n = 2048 / BLOCK_N;
    if (ag != nullptr && ag->world > 1) {
        if (kMajorB != 0 || p.batch != 1) throw std::runtime_error("gemm: AG fusion needs a K-major, un-batched B");
        if (static_cast<int64_t>(ag->rows_per_slab) * K * 2 != ag->slab_bytes || ag->slab_bytes % 16 != 0)
            throw std::runtime_error("gemm: AG fusion needs whole rows per slab");
        p.ag = *ag;
        p.n_rot = static_cast<int>((static_cast<int64_t>(ag->rank) * ag->rows_per_slab) / BLOCK_N) % p.n_tiles;
        cudaMemsetAsync(ag->flags, 0, sizeof(uint32_t) * (ag->world + 1), stream);  // slab counters + chunk counter
    }
    const int64_t total = static_cast<int64_t>(p.m_units) * p.n_tiles * p.batch;
    int units = resident_units;
    if (max_ctas > 0) units = std::min(units, max_ctas / kClusterM);  // max_ctas >= kClusterM (gemm_bf16)
    units = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(total, units)));
    cfg.gridDim = dim3(units * kClusterM);
    check(cudaLaunchKernelEx(&cfg, kern, ta, tb, td, tx, p), "gemm launch failed");
    check(cudaGetLastError(), "gemm launch failed");
}

// SwiGLU epilogues: the checks that keep them within what the kernel implements, each named in its message.
void gemm_glu(const GemmOperand& A, int major_a, const GemmOperand& B, int major_b, const GemmOperand& D,
              const GemmOperand* aux_out, int M, int N, int K, const GemmEpilogue& epi, int block_n, int cluster,
              int max_ctas, cudaStream_t stream, const GemmAgFuse* ag) {
    const bool fwd = epi.act == kActSwiglu;
    if (epi.residual != nullptr) throw std::runtime_error("gemm: SwiGLU epilogues take no residual");
    if (epi.row_scale != nullptr) throw std::runtime_error("gemm: SwiGLU epilogues take no row_scale");
    if (A.nb_inner * A.nb_outer > 1 || B.nb_inner * B.nb_outer > 1 || D.nb_inner * D.nb_outer > 1)
        throw std::runtime_error("gemm: SwiGLU epilogues take no batched operands");
    if (ag != nullptr && ag->world > 1) throw std::runtime_error("gemm: SwiGLU epilogues take no AG fusion");
    if (N % 8 != 0) throw std::runtime_error("gemm: SwiGLU needs N = H' = Hd / 2 to be a multiple of 8 (Hd % 16 == 0)");
    if (fwd) {
        if (major_a != 0 || major_b != 0) throw std::runtime_error("gemm: SwiGLU forward needs K-major A and B");
        if (epi.aux_in != nullptr || epi.colsum != nullptr)
            throw std::runtime_error("gemm: SwiGLU forward takes no aux_in and no column sums");
        if (epi.has_aux_out != (aux_out != nullptr))
            throw std::runtime_error("gemm: SwiGLU forward: has_aux_out and the aux output go together");
    } else {
        if (major_a != 0 || major_b != 1) throw std::runtime_error("gemm: dSwiGLU needs K-major A and MN-major B");
        if (epi.aux_in == nullptr || aux_out == nullptr || !epi.has_aux_out)
            throw std::runtime_error("gemm: dSwiGLU needs aux_in (u) and an aux output (du_val)");
        if (epi.bias != nullptr) throw std::runtime_error("gemm: dSwiGLU takes no bias");
    }
    if (block_n == 0) block_n = 256;
    if (block_n != 128 && block_n != 256) throw std::runtime_error("gemm: SwiGLU block_n must be 128 or 256");
    if (cluster == 0 || max_ctas == 1) cluster = 1;
#define B200_GLU(MB, BN, ST, ACT)                                                                            \
    cluster == 2 ? launch<0, MB, BN, ST, 2, false, ACT>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag) \
                 : launch<0, MB, BN, ST, 1, false, ACT>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag)
    if (fwd)
        block_n == 256 ? B200_GLU(0, 256, 4, kActSwiglu) : B200_GLU(0, 128, 6, kActSwiglu);
    else
        block_n == 256 ? B200_GLU(1, 256, 4, kActDSwiglu) : B200_GLU(1, 128, 6, kActDSwiglu);
#undef B200_GLU
}

}  // namespace

CUtensorMap make_tensor_map_4d(const GemmOperand& op, int64_t inner, int64_t outer, int box_inner, int box_outer,
                               int swizzle_bytes) {
    return make_tmap(op, inner, outer, box_inner, box_outer, swizzle_bytes);
}

void gemm_bf16(const GemmOperand& A, int major_a, const GemmOperand& B, int major_b, const GemmOperand& D,
               const GemmOperand* aux_out, int M, int N, int K, const GemmEpilogue& epi, int block_n, int cluster,
               int max_ctas, cudaStream_t stream, const GemmAgFuse* ag) {
    if (epi.act == kActSwiglu || epi.act == kActDSwiglu) {
        gemm_glu(A, major_a, B, major_b, D, aux_out, M, N, K, epi, block_n, cluster, max_ctas, stream, ag);
        return;
    }
    if (N % 8 != 0 && (epi.residual || epi.aux_in))
        throw std::runtime_error("gemm: N must be a multiple of 8 when residual/aux_in are used");
    if (epi.act == kActDGelu && (epi.residual != nullptr || epi.aux_in == nullptr))
        throw std::runtime_error("gemm: dGELU epilogue needs aux_in and cannot be combined with a residual");
    if (D.nb_inner * D.nb_outer > 1 && (epi.bias || epi.residual || epi.aux_in))
        throw std::runtime_error("gemm: bias/residual/aux_in are not supported for batched problems");
    if (cluster != 0 && cluster != 1 && cluster != 2) throw std::runtime_error("gemm: cluster must be 0 (auto), 1 or 2");
    if (block_n == 0) block_n = (N > 128) ? 256 : 128;
    // Auto is one CTA per tile: CTA pairs are no faster on the ViT-10B block GEMMs (measurements in DESIGN.md).
    if (cluster == 0 || max_ctas == 1) cluster = 1;
    if (epi.row_scale != nullptr) {  // the forward of a linear layer: instantiated for K-major A and B only
        if (epi.rows_per_scale < 1) throw std::runtime_error("gemm: row_scale needs rows_per_scale >= 1");
        if (epi.act != kActNone || epi.has_aux_out || aux_out != nullptr || epi.colsum != nullptr ||
            D.nb_inner * D.nb_outer > 1)
            throw std::runtime_error("gemm: row_scale only with no activation, no aux output, no column sums, unbatched");
        if (major_a != 0 || major_b != 0) throw std::runtime_error("gemm: row_scale needs K-major A and B");
        if (block_n == 256)
            cluster == 2 ? launch<0, 0, 256, 4, 2, true>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag)
                         : launch<0, 0, 256, 4, 1, true>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag);
        else if (block_n == 128)
            cluster == 2 ? launch<0, 0, 128, 6, 2, true>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag)
                         : launch<0, 0, 128, 6, 1, true>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag);
        else
            throw std::runtime_error("gemm: unsupported block_n");
        return;
    }
#define B200_DISPATCH(MA, MB, BN, ST)                                                             \
    if (major_a == MA && major_b == MB && block_n == BN) {                                        \
        if (cluster == 2)                                                                         \
            launch<MA, MB, BN, ST, 2>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag);      \
        else                                                                                      \
            launch<MA, MB, BN, ST, 1>(A, B, D, aux_out, M, N, K, epi, max_ctas, stream, ag);      \
        return;                                                                                   \
    }
    B200_DISPATCH(0, 0, 256, 4)
    B200_DISPATCH(0, 1, 256, 4)
    B200_DISPATCH(1, 1, 256, 4)
    B200_DISPATCH(1, 0, 256, 4)
    B200_DISPATCH(0, 0, 128, 6)
    B200_DISPATCH(0, 1, 128, 6)
    B200_DISPATCH(1, 1, 128, 6)
    B200_DISPATCH(1, 0, 128, 6)
#undef B200_DISPATCH
    throw std::runtime_error("gemm: unsupported (major_a, major_b, block_n) combination");
}

}  // namespace b200
