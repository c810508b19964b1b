// Host API of the LayerScale kernels (layer_scale.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

// LayerScale folded into a linear layer: W [D, K] and every other matrix contiguous row-major bf16; b / gamma bf16 [D].
// Forward: Wg = bf16(gamma_c * W[c, :]) and bg = bf16(gamma_c * b_c).
void layer_scale_fold(const __nv_bfloat16* W, const __nv_bfloat16* b, const __nv_bfloat16* gamma, __nv_bfloat16* Wg,
                      __nv_bfloat16* bg, int64_t D, int64_t K, cudaStream_t stream);
// Backward: dW holds M = dy'^T a (the wgrad of the un-scaled weight) on entry and bf16(gamma_c * M[c, :]) on exit;
// S fp32 [D] = column sums of dy'.  Writes Wg as the forward does, db_c = gamma_c S_c and
// dgamma_c = sum_k W[c, k] M[c, k] + b_c S_c (fp32 [D], overwritten, one CTA per row: no atomics, deterministic).
void layer_scale_bwd(const __nv_bfloat16* W, const __nv_bfloat16* b, const __nv_bfloat16* gamma, __nv_bfloat16* dW,
                     const float* S, __nv_bfloat16* Wg, float* db, float* dgamma, int64_t D, int64_t K,
                     cudaStream_t stream);

}  // namespace b200
