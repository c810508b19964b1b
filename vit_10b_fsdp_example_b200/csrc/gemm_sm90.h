// Host API of the sm_90a wgmma GEMM (see gemm_sm90.cu).
// Every nn.Linear / conv-as-GEMM / attention matmul of the reference model (run_vit_training.py:124-153 via timm) runs on it.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

enum GemmAct : int { kActNone = 0, kActGelu = 1, kActDGelu = 2, kActSwiglu = 3, kActDSwiglu = 4 };

// SwiGLU epilogues (timm SwiGLUPacked: u = [gate | value], g = silu(gate) * value), with N = H' = Hd / 2 output columns:
//   kActSwiglu   forward, K-major A and B.  B is the whole [Hd, K] fc1 weight and bias the whole [Hd] fc1 bias; a tile
//                multiplies by B rows [n, n + BLOCK_N / 2) (gate) and [H' + n, ...) (value) and writes
//                D[m, n] = silu(a) * b, a / b the gate / value pre-activations with bias.  With an aux output (the
//                [M, Hd] matrix u) it also stores a at u[m, n] and b at u[m, H' + n].
//   kActDSwiglu  fc2 dgrad, K-major A, MN-major B: acc = dh[m, n]; aux_in = u [M, Hd] (a at column n, b at H' + n).
//                Writes du_gate = dh * b * silu'(a) through D (columns [0, H') of du) and du_val = dh * silu(a) through
//                the aux output (columns [H', Hd) of du); colsum [Hd] receives the column sums of both halves.
// Neither takes a residual, a row scale, batched operands or AG fusion; H' must be a multiple of 8 (Hd % 16 == 0).

// A strided bf16 matrix with up to two batch dimensions.  `ld` and the batch strides are in elements.
// The *inner* (contiguous) extent and the *outer* extent are implied by the GEMM shape and the major.
struct GemmOperand {
    const void* ptr = nullptr;
    int64_t ld = 0;
    int64_t nb_inner = 1, stride_b_inner = 0;
    int64_t nb_outer = 1, stride_b_outer = 0;
};

struct GemmEpilogue {
    const __nv_bfloat16* bias = nullptr;      // [N]           v += bias[n]
    const __nv_bfloat16* residual = nullptr;  // [M, ld_res]   v += residual[m, n]   (after activation)
    const __nv_bfloat16* aux_in = nullptr;    // [M, ld_aux]   pre-activation for kActDGelu / kActDSwiglu
    float* colsum = nullptr;                  // [N] fp32      atomically += sum_m out[m, n]
    int64_t ld_res = 0;
    int64_t ld_aux = 0;
    int64_t colsum_bi_stride = 0;
    int res_row_mod = 0;  // > 0: residual row = m % res_row_mod (broadcast a [rows, N] table, e.g. pos_embed)
    int act = kActNone;
    int has_aux_out = 0;  // also store the pre-activation (after bias) through the aux tensor map
    // [ceil(M / rows_per_scale)] fp32: v = (acc + bias) * row_scale[m / rows_per_scale], before the residual add.
    // Per-sample scales of stochastic depth (rows_per_scale = tokens per image).  Only with kActNone, no aux output,
    // no column sums and unbatched problems.
    const float* row_scale = nullptr;
    int rows_per_scale = 0;
};

// All-gather fused into the GEMM (B operand = an FSDP-sharded weight, rank r owns rows [r*rows_per_slab, ...)):
// a spare warp of every CTA pulls the peers' slabs over NVLink (P2P loads from symmetric memory) straight into the
// local gathered buffer and bumps a per-slab counter; the TMA producer waits for the slab(s) a tile needs, and tiles
// are visited in slab-arrival order (own slab first), so the tensor cores start after 1/W of the weight is there
// and the transfer of the rest hides under the math.  No NCCL, no host sync, no separate gather kernel.
struct GemmAgFuse {
    int world = 0;            // 0/1 = disabled
    int rank = 0;
    int rows_per_slab = 0;    // B rows (output features) owned by each rank
    int64_t slab_bytes = 0;   // bytes per slab
    uint64_t peer_src[16] = {0};  // per rank: address of its slab (peer-mapped symmetric memory)
    void* dst = nullptr;      // local gathered B (slab r lands at dst + r * slab_bytes)
    uint32_t* flags = nullptr;  // [world] device counters; zeroed by gemm_bf16 before the launch
};

// D[b][M, N] = epi(A[b] (M x K) * B[b] (N x K)^T).  major_x: 0 = K contiguous, 1 = M/N contiguous.
// block_n: 0 = auto, else 128 / 256.  cluster: 0 = auto (= 1), 1 = one CTA per tile, 2 = CTA pairs along M sharing
// B through TMA multicast (1 is used when max_ctas = 1).  max_ctas: 0 = all SMs (used to carve SMs out for comm kernels).
// With N % 8 != 0 the TMA store writes whole 16-byte units, so the columns [N, pad8(N)) of every row are written too:
// with +0 in D, with unspecified values in the aux output.  Every ld is a multiple of 8, so this stays inside the row,
// but a D or aux output that is a column slice of a wider matrix must leave those columns to the GEMM.
void gemm_bf16(const GemmOperand& A, int major_a, const GemmOperand& B, int major_b, const GemmOperand& D,
               const GemmOperand* aux_out, int M, int N, int K, const GemmEpilogue& epi, int block_n, int cluster,
               int max_ctas, cudaStream_t stream, const GemmAgFuse* ag = nullptr);

// Cached 4-D bf16 TMA descriptor: dims (inner, outer, op.nb_inner, op.nb_outer), box (box_inner, box_outer, 1, 1).
CUtensorMap make_tensor_map_4d(const GemmOperand& op, int64_t inner, int64_t outer, int box_inner, int box_outer,
                               int swizzle_bytes);

}  // namespace b200
