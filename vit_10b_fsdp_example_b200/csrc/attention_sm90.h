// Host API of the fused wgmma attention kernels (attention_sm90.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

// Even N, head dim 64 / 128 / 160.
bool attention_supported(int N, int hd);

// qkv: packed [B*N, 3*H*hd] (row stride ld_qkv).  out: [B*N, H*hd].  lse: [B*H, N] fp32 or null.
// probs: normalised softmax [B*H, N, ldp] bf16 or null (only written when the un-fused backward needs it).
void attention_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, __nv_bfloat16* probs,
                   int64_t ldp, int B, int N, int H, int hd, cudaStream_t stream);

// Fused backward.  dout / out: [B*N, H*hd] gradient and forward output of the attention core, lse: [B*H, N] from the
// forward, delta: [B*H, N] fp32 workspace (written here), dqkv: packed [B*N, 3*H*hd].
// colsum (optional): zero-initialised fp32 [3 * D]; receives the column sums of dq | dk | dv (the qkv bias gradient)
// straight from the epilogue tiles.
void attention_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                   const __nv_bfloat16* out, int64_t ld_o, const float* lse, float* delta, __nv_bfloat16* dqkv,
                   int B, int N, int H, int hd, cudaStream_t stream, float* colsum = nullptr);

}  // namespace b200
