// Host API of the fused wgmma attention kernels (attention_sm90.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

// Whether the model routes (N, hd) through the fused kernels: even N and head dim 32, 40, 48, 64, 128 or 160.  The
// kernels themselves also take hd 72, 80, 88, 96, 104, 112, 136 and 144 (attention_sm90.cu says why those are not
// routed); attention_fwd / attention_bwd throw on any other head dim.
bool attention_supported(int N, int hd);

// Whether the kernels take (N, hd) at all: even N >= 2 and a head dim listed above (attention_fwd / attention_bwd throw
// otherwise).
bool attention_shape_ok(int N, int hd);

// qkv: packed [B*N, 3*H*hd] (row stride ld_qkv).  out: [B*N, H*hd].  lse: [B*H, N] fp32 or null.
// probs: normalised softmax [B*H, N, ldp] bf16 or null (only written when the un-fused backward needs it).
// drop_p > 0: attention dropout with the mask the dropout kernel (dropout.cuh) draws for key drop_key over the
// probabilities laid out as [B*H, N, pad8(N)]; lse stays that of the undropped scores, probs must be null.
void attention_fwd(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, __nv_bfloat16* probs,
                   int64_t ldp, int B, int N, int H, int hd, cudaStream_t stream, float drop_p = 0.f,
                   uint64_t drop_key = 0);

// Fused backward.  dout / out: [B*N, H*hd] gradient and forward output of the attention core, lse: [B*H, N] from the
// forward, delta: [B*H, N] fp32 workspace (written here), dqkv: packed [B*N, 3*H*hd].
// colsum (optional): zero-initialised fp32 [3 * D]; receives the column sums of dq | dk | dv (the qkv bias gradient)
// straight from the epilogue tiles.  drop_p / drop_key: those of the forward.
void attention_bwd(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                   const __nv_bfloat16* out, int64_t ld_o, const float* lse, float* delta, __nv_bfloat16* dqkv,
                   int B, int N, int H, int hd, cudaStream_t stream, float* colsum = nullptr, float drop_p = 0.f,
                   uint64_t drop_key = 0);

// The attention-dropout kernels (attention_drop_sm90.cu); attention_fwd / attention_bwd dispatch to them when
// drop_p != 0.  attention_bwd_drop expects delta already computed by attention_bwd's delta kernel.
void attention_fwd_drop(const __nv_bfloat16* qkv, int64_t ld_qkv, __nv_bfloat16* out, float* lse, int B, int N, int H,
                        int hd, float drop_p, uint64_t drop_key, cudaStream_t stream);
void attention_bwd_drop(const __nv_bfloat16* qkv, int64_t ld_qkv, const __nv_bfloat16* dout, int64_t ld_do,
                        const float* lse, const float* delta, __nv_bfloat16* dqkv, int B, int N, int H, int hd,
                        float* colsum, float drop_p, uint64_t drop_key, cudaStream_t stream);

}  // namespace b200
