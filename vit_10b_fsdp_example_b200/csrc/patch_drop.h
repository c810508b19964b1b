// Host API of the patch-dropout kernels (patch_drop.cu): timm's PatchDropout(prob=R, num_prefix_tokens=P, ordered=True)
// in training, every image keeping K = max(1, int(N * (1 - R))) of its N patch tokens.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

#include "elementwise.h"

namespace b200 {

constexpr int kPatchDropMaxN = 4096;  // a 64 x 64 patch grid: the select kernel sorts one image's keys in shared memory

// keep [B, K] int32: the kept patches of image g = offset + b in ascending patch order, namely the K patches with the
// smallest (r, n), r = word n % 4 of philox4x32_10(n / 4, g, key).  inv [B, N] int32: the row of patch n in image b's
// kept list, or -1 when the patch is dropped.  1 <= K <= N <= kPatchDropMaxN, offset + B <= 2^32.
void patch_drop_select(int* keep, int* inv, int64_t B, int64_t N, int64_t K, int64_t offset, uint64_t key,
                       cudaStream_t stream);
// The patch im2col of the kept patches only: cols [B * K, Kpad] bf16, row b * K + i is patch keep[b * K + i] of image b,
// with the batch mixing of ``im2col`` (applied per pixel before the selection).  keep as patch_drop_select writes it.
void im2col_gather(const void* img, bool img_is_bf16, const int* keep, __nv_bfloat16* cols, int B, int S, int P,
                   int Kpad, int K, cudaStream_t stream, const Im2colMix& mix = Im2colMix());
// out [rows, D] = pos[keep[r]] for every row r (rows = B * K); pos [N, D]; D % 8 == 0, all 16-byte aligned.
void pos_gather(const __nv_bfloat16* pos, const int* keep, __nv_bfloat16* out, int64_t rows, int64_t D,
                cudaStream_t stream);
// Backward of the kept-token assembly.  dx0 [B * (P + K), D]; dtok [P + N, D] fp32 (overwritten): dtok[j] for a prefix
// row j < P is sum_b dx0[b, j], for patch n it is the sum of dx0[b, P + inv[b, n]] over the images that kept patch n
// (zero when none did), added in b order: no atomics, the same bits in every run.  dpatch [B * K, D] (may be null)
// receives the patch rows of dx0 as one contiguous matrix, the patch-embed wgrad operand.
void patch_drop_bwd(const __nv_bfloat16* dx0, const int* inv, __nv_bfloat16* dpatch, float* dtok, int64_t B,
                    int64_t N, int64_t K, int64_t P, int64_t D, cudaStream_t stream);

}  // namespace b200
