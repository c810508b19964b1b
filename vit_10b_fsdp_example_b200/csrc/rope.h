// Host API of the rotary position embedding kernels (rope.cu) and of the RoPE-fused QK normalisation (qk_norm.cu).
//
// 2-D axial RoPE (EVA-02, timm RotaryEmbeddingCat) on the packed [rows, 3D] qkv buffer, D = H * hd, rows = B * tokens.
// Pair i of a q or k head is its interleaved elements (2i, 2i + 1); it is rotated by the angle whose cosine and sine
// are cos[n, i] / sin[n, i], where n is the patch's row of the fp32 [n_tab, hd / 2] tables:
//     y0 = x0 * cos - x1 * sin,  y1 = x1 * cos + x0 * sin      (the backward applies the transpose R^T).
// Token j of image b is a prefix token (class / register) for j < prefix, left as it is; otherwise its table row is
// keep[b, j - prefix] (patch dropout: the kept patch's original index) or, without keep, j - prefix.
// hd % 8 == 0 and 8 <= hd <= 256; every matrix 16-byte aligned with ld % 8 == 0 and ld >= 3D.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

struct RopeArgs {
    const float* cos = nullptr;  // fp32 [n_tab, hd / 2]; null = no rotation
    const float* sin = nullptr;
    const int* keep = nullptr;   // int32 [B, tokens - prefix] or null
    int tokens = 0;              // tokens per image (P + K under patch dropout)
    int prefix = 0;              // P: class and register tokens, not rotated
    int n_tab = 0;               // table rows (the patches of the full grid)
};

// Throws std::runtime_error naming the check ("<what>: ...") for a head dim outside [8, 256] or not a multiple of 8, a
// bad B / H / tokens / prefix, B * tokens past 32 bits, unaligned tables, or tables with fewer rows than patch tokens.
// The values of keep are not checked: they must be in [0, n_tab).
void check_rope_args(const char* what, const RopeArgs& rope, int B, int H, int hd);

// out[:, 0:2D) = R qkv[:, 0:2D).  out == qkv (ld_out == ld) works in place and leaves the v columns alone; a separate
// out gets a bit-exact copy of v and of the prefix rows.
void rope_fwd(const __nv_bfloat16* qkv, int64_t ld, __nv_bfloat16* out, int64_t ld_out, const RopeArgs& rope, int B,
              int H, int hd, cudaStream_t stream);
// In place on dqkv[:, 0:2D): dq / dk become R^T dq / R^T dk (dv is not touched).  colsum fp32 [2D] is atomically
// added the column sums of the stored bf16 dq / dk, prefix rows included: zero it first.
void rope_bwd(__nv_bfloat16* dqkv, int64_t ld, const RopeArgs& rope, int B, int H, int hd, float* colsum,
              cudaStream_t stream);

// QK normalisation followed by the rotation, rounded to bf16 once (qk_norm_fwd of elementwise.h, then R in fp32).
void qk_norm_rope_fwd(const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq, const __nv_bfloat16* bq,
                      const __nv_bfloat16* wk, const __nv_bfloat16* bk, __nv_bfloat16* out, int64_t ld_out,
                      float* mean, float* rstd, const RopeArgs& rope, int B, int H, int hd, float eps,
                      cudaStream_t stream);
// Its backward: R^T on the incoming dq / dk in registers, then qk_norm_bwd's LayerNorm backward, dw / db and column
// sums (the q / k part of the qkv bias gradient).
void qk_norm_rope_bwd(__nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* qkv, int64_t ld,
                      const __nv_bfloat16* wq, const __nv_bfloat16* wk, const float* mean, const float* rstd,
                      float* dwq, float* dbq, float* dwk, float* dbk, float* colsum, const RopeArgs& rope, int B,
                      int H, int hd, cudaStream_t stream);

}  // namespace b200
