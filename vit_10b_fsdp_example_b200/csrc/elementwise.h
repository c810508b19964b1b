// Host API of the memory-bound sm_90a kernels (see elementwise.cu).
// LayerNorm, softmax, GELU, cross-entropy, AdamW, clipping: the ATen/XLA ops behind run_vit_training.py:134-162,229,237,270.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace b200 {

void layernorm_fwd(const __nv_bfloat16* x, const __nv_bfloat16* gamma, const __nv_bfloat16* beta, __nv_bfloat16* y,
                   float* mean, float* rstd, int rows, int D, float eps, cudaStream_t stream);

// dgamma / dbeta / dxsum are fp32 [D] accumulators (atomically added to; zero them first).
void layernorm_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                   const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                   float* dxsum, int rows, int D, cudaStream_t stream);

void softmax_fwd(__nv_bfloat16* s, int64_t rows, int n, int64_t ld, float scale, cudaStream_t stream);
void softmax_bwd(__nv_bfloat16* dp, const __nv_bfloat16* p, int64_t rows, int n, int64_t ld, float scale,
                 cudaStream_t stream);

// loss (fp32 scalar, atomically added) = mean CE; dlogits may be null (eval); correct may be null (counts argmax ==
// target).  lam < 1 mixes row b's target with that of row B-1-b (B even); smoothing > 0 smooths both (timm
// mixup_target): the soft target is lam * smooth(y_b) + (1 - lam) * smooth(y_{B-1-b}).
void cross_entropy(const __nv_bfloat16* logits, const int64_t* target, __nv_bfloat16* dlogits, float* loss,
                   int* correct, int B, int C, cudaStream_t stream, double lam = 1.0, double smoothing = 0.0);

// Batch mixing fused into im2col (timm Mixup, mode 'batch'): image b is mixed with image B-1-b (B even).
struct Im2colMix {
    int mode = 0;               // 0 none, 1 Mixup (blend with lam / mlam), 2 CutMix (the box comes from image B-1-b)
    float lam = 1.f, mlam = 0.f;  // Mixup weights: fp32(lam) and fp32(1 - lam), 1 - lam taken in double
    int yl = 0, yh = 0, xl = 0, xh = 0;  // CutMix box [yl, yh) x [xl, xh) in pixels
};
void im2col(const void* img, bool img_is_bf16, __nv_bfloat16* cols, int B, int S, int P, int Kpad,
            cudaStream_t stream, const Im2colMix& mix = Im2colMix());

// Wide-row LayerNorm backward as a cp.async.bulk row pipeline (layernorm_stream.cu); same contract as layernorm_bwd.
bool layernorm_bwd_stream_supported(int D);
void layernorm_bwd_stream(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* gamma, const float* mean,
                          const float* rstd, const __nv_bfloat16* dres, __nv_bfloat16* dx, float* dgamma, float* dbeta,
                          float* dxsum, int rows, int D, cudaStream_t stream);
void gelu_fwd(const __nv_bfloat16* u, __nv_bfloat16* g, int64_t n, cudaStream_t stream);
void dgelu_mul(const __nv_bfloat16* dg, const __nv_bfloat16* u, __nv_bfloat16* du, int64_t n, cudaStream_t stream);
// SwiGLU on a packed u = [gate | value] [M, hidden] (row-major, hidden % 16 == 0, 16-byte aligned):
// g [M, hidden / 2] = silu(gate) * value;  du [M, hidden] = [dg * value * silu'(gate) | dg * silu(gate)].
void swiglu_fwd(const __nv_bfloat16* u, __nv_bfloat16* g, int64_t M, int64_t hidden, cudaStream_t stream);
void swiglu_bwd(const __nv_bfloat16* dg, const __nv_bfloat16* u, __nv_bfloat16* du, int64_t M, int64_t hidden,
                cudaStream_t stream);
// y = x * keep / (1 - p), keep = Philox-4x32-10(key, vector index): a pure function of (key, position), so recompute and
// backward regenerate the mask.  p is quantised to 1/65536.  y may alias x.
void dropout(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, float p, uint64_t key, cudaStream_t stream);
// Stochastic depth: scale[b] = dropout_scale or 0 for sample sample_offset + b, drawn from the dropout kernel's Philox
// stream (keep bit g % 8 of vector g / 8).  Effective keep probability 1 - thresh16(p) / 65536.
void drop_path_scale(float* scale, int B, int64_t sample_offset, float p, uint64_t key, cudaStream_t stream);
// dt[r, :] = bf16(scale[r / N] * dy[r, :]); colsum (fp32 [C], atomically added to: zero it first) += column sums of dt.
void drop_path_bwd(const __nv_bfloat16* dy, const float* scale, __nv_bfloat16* dt, float* colsum, int64_t rows, int C,
                   int N, cudaStream_t stream);
// pooled[b] = mean over the N tokens of image b; backward broadcasts dpooled[b] / N to every token row.
void meanpool_fwd(const __nv_bfloat16* xn, __nv_bfloat16* pooled, int B, int N, int D, cudaStream_t stream);
void meanpool_bwd(const __nv_bfloat16* dpooled, __nv_bfloat16* dxn, int B, int N, int D, cudaStream_t stream);
void colsum(const __nv_bfloat16* x, float* out, int64_t rows, int C, cudaStream_t stream);

// QK normalisation (qk_norm.cu) on the packed [T, 3D] qkv buffer, D = H * hd, hd % 8 == 0 and 8 <= hd <= 256.
// Forward: out[:, 0:2D) = LayerNorm over hd of each q head (wq, bq) and k head (wk, bk); mean / rstd fp32 [T, 2, H].
// out == qkv (ld_out == ld) works in place and leaves the v columns alone; a separate out gets a copy of them.
void qk_norm_fwd(const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq, const __nv_bfloat16* bq,
                 const __nv_bfloat16* wk, const __nv_bfloat16* bk, __nv_bfloat16* out, int64_t ld_out, float* mean,
                 float* rstd, int T, int H, int hd, float eps, cudaStream_t stream);
// Backward, in place on dqkv[:, 0:2D) (the gradient of the normalised q / k in, of the un-normalised q / k out; the dv
// columns are not touched).  dwq / dbq / dwk / dbk fp32 [hd] and colsum fp32 [2D] (column sums of the new bf16 dq / dk)
// are atomically added to: zero them first.
void qk_norm_bwd(__nv_bfloat16* dqkv, int64_t ld_d, const __nv_bfloat16* qkv, int64_t ld, const __nv_bfloat16* wq,
                 const __nv_bfloat16* wk, const float* mean, const float* rstd, float* dwq, float* dbq, float* dwk,
                 float* dbk, float* colsum, int T, int H, int hd, cudaStream_t stream);
void sumsq(const void* x, bool is_bf16, int64_t n, float* out, cudaStream_t stream);

// hyper (optional, device): [lr, step] override the host values (CUDA-graph friendly)
// ema_hi / ema_lo (optional, both or neither): the model EMA in split form, updated in the same pass as
// ema = fmaf(ema_decay, ema, (1 - ema_decay) * w) from the new master w; null = no EMA (the plain kernel)
void adamw_split(uint16_t* hi, int16_t* lo, float* m, float* v, const void* grad, bool grad_is_bf16, int64_t n,
                 const float* clip_coef, float lr, float beta1, float beta2, float eps, float wd, int step,
                 cudaStream_t stream, const float* hyper = nullptr, uint16_t* ema_hi = nullptr,
                 int16_t* ema_lo = nullptr, float ema_decay = 0.f);
// ema (optional): fp32 model EMA, same recurrence
void adamw_fp32(float* w, float* m, float* v, const void* grad, bool grad_is_bf16, int64_t n, const float* clip_coef,
                float lr, float beta1, float beta2, float eps, float wd, int step, cudaStream_t stream,
                float* ema = nullptr, float ema_decay = 0.f);
void split_fp32(const float* w, uint16_t* hi, int16_t* lo, int64_t n, cudaStream_t stream);
void merge_fp32(const uint16_t* hi, const int16_t* lo, float* w, int64_t n, cudaStream_t stream);
void clip_coef(const float* sumsq_in, float max_norm, float* coef, float* norm_out, cudaStream_t stream);

}  // namespace b200
