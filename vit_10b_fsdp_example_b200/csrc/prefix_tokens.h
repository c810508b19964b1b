// Host API of the prefix-token kernels (prefix_tokens.cu): the class token and register tokens of timm's
// VisionTransformer(class_token=True, reg_tokens=R), P = 1 + R rows placed in front of every image's N patch rows.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

// x0 [B * T, D] (T = N + P) from the patch rows y [B * N, D] (patch GEMM output, bias and patch position rows already
// added): row b * T + j is y[b * N + j - P] for j >= P and bf16(prefix[j] + pos[j]) for j < P, summed in fp32 and
// rounded once, where prefix[0] = cls [D] and prefix[1 + r] = reg[r] (reg [P - 1, D], may be null when P == 1).
// pos [P, D] may be null (prefix tokens without a position embedding).  All buffers contiguous, 16-byte aligned,
// D % 8 == 0.
void tokens_fwd(const __nv_bfloat16* y, const __nv_bfloat16* cls, const __nv_bfloat16* reg, const __nv_bfloat16* pos,
                __nv_bfloat16* x0, int64_t B, int64_t N, int64_t P, int64_t D, cudaStream_t stream);
// One pass over dx0 [B * T, D]: dpatch [B * N, D] receives the patch rows (the patch-embed wgrad operand) and
// dtok [T, D] fp32 (overwritten) the per-token sums over the batch, dtok[j] = sum_b dx0[b * T + j], added in b order
// by one thread per 8 columns of row j: no atomics, the same bits in every run.
void tokens_bwd(const __nv_bfloat16* dx0, __nv_bfloat16* dpatch, float* dtok, int64_t B, int64_t N, int64_t P,
                int64_t D, cudaStream_t stream);

}  // namespace b200
