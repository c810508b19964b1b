// pybind11 / ATen bindings for the sm_90a kernels.  Compiled by g++ (no CUDA device code here), so the
// .cu files stay free of the heavy torch headers and rebuild in seconds.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cmath>
#include <optional>
#include <vector>

#include "attention_sm90.h"
#include "comm.h"
#include "elementwise.h"
#include "gemm_sm90.h"
#include "layer_scale.h"
#include "patch_drop.h"
#include "prefix_tokens.h"

namespace {

using torch::Tensor;
using OptT = std::optional<Tensor>;

inline const __nv_bfloat16* bf16_ptr(const Tensor& t) {
    TORCH_CHECK(t.is_cuda(), "expected a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == at::kBFloat16, "expected a bf16 tensor");
    return reinterpret_cast<const __nv_bfloat16*>(t.data_ptr());
}
inline __nv_bfloat16* bf16_mut(Tensor& t) { return const_cast<__nv_bfloat16*>(bf16_ptr(t)); }
inline float* f32_ptr(const Tensor& t) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat, "expected a CUDA fp32 tensor");
    return reinterpret_cast<float*>(t.data_ptr());
}
inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// batch = [] or [nb_inner, nb_outer, a_sbi, a_sbo, b_sbi, b_sbo, d_sbi, d_sbo] (strides in elements)
void gemm(Tensor a, int64_t lda, int64_t major_a, Tensor b, int64_t ldb, int64_t major_b, Tensor d, int64_t ldd,
          int64_t M, int64_t N, int64_t K, OptT bias, OptT residual, int64_t ld_res, int64_t res_row_mod, OptT aux_in,
          int64_t ld_aux, OptT aux_out, int64_t ld_aux_out, OptT colsum, int64_t colsum_bi_stride, int64_t act,
          std::vector<int64_t> batch, int64_t block_n, int64_t cluster, int64_t max_ctas, std::vector<int64_t> ag,
          OptT row_scale, int64_t rows_per_scale) {
    c10::cuda::CUDAGuard guard(a.device());
    b200::GemmOperand A, B, D, X;
    A.ptr = bf16_ptr(a), A.ld = lda;
    B.ptr = bf16_ptr(b), B.ld = ldb;
    D.ptr = bf16_ptr(d), D.ld = ldd;
    if (!batch.empty()) {
        TORCH_CHECK(batch.size() == 8, "batch spec must have 8 entries");
        A.nb_inner = B.nb_inner = D.nb_inner = batch[0];
        A.nb_outer = B.nb_outer = D.nb_outer = batch[1];
        A.stride_b_inner = batch[2], A.stride_b_outer = batch[3];
        B.stride_b_inner = batch[4], B.stride_b_outer = batch[5];
        D.stride_b_inner = batch[6], D.stride_b_outer = batch[7];
    }
    b200::GemmEpilogue e;
    if (bias.has_value()) e.bias = bf16_ptr(*bias);
    if (residual.has_value()) e.residual = bf16_ptr(*residual), e.ld_res = ld_res, e.res_row_mod = (int)res_row_mod;
    if (aux_in.has_value()) e.aux_in = bf16_ptr(*aux_in), e.ld_aux = ld_aux;
    if (colsum.has_value()) e.colsum = f32_ptr(*colsum), e.colsum_bi_stride = colsum_bi_stride;
    e.act = static_cast<int>(act);
    if (row_scale.has_value()) {
        TORCH_CHECK(row_scale->is_contiguous() && row_scale->numel() * rows_per_scale >= M,
                    "gemm: row_scale must be contiguous with one entry per rows_per_scale rows");
        e.row_scale = f32_ptr(*row_scale), e.rows_per_scale = (int)rows_per_scale;
    }
    if (aux_out.has_value()) {
        X = D;
        X.ptr = bf16_ptr(*aux_out), X.ld = ld_aux_out;
        e.has_aux_out = 1;
    }
    // ag = [] or [world, rank, rows_per_slab, slab_bytes, dst_ptr, flags_ptr, peer_src_0, ..., peer_src_{W-1}]
    b200::GemmAgFuse fuse;
    if (!ag.empty()) {
        TORCH_CHECK(ag.size() >= 6 && (int64_t)ag.size() == 6 + ag[0] && ag[0] <= 16, "bad AG-fusion spec");
        fuse.world = (int)ag[0], fuse.rank = (int)ag[1], fuse.rows_per_slab = (int)ag[2], fuse.slab_bytes = ag[3];
        fuse.dst = reinterpret_cast<void*>(ag[4]);
        fuse.flags = reinterpret_cast<uint32_t*>(ag[5]);
        for (int64_t r = 0; r < ag[0]; ++r) fuse.peer_src[r] = static_cast<uint64_t>(ag[6 + r]);
    }
    b200::gemm_bf16(A, (int)major_a, B, (int)major_b, D, aux_out.has_value() ? &X : nullptr, (int)M, (int)N, (int)K, e,
                    (int)block_n, (int)cluster, (int)max_ctas, cur_stream(), ag.empty() ? nullptr : &fuse);
}

void layernorm_fwd(Tensor x, Tensor gamma, Tensor beta, Tensor y, Tensor mean, Tensor rstd, double eps) {
    c10::cuda::CUDAGuard guard(x.device());
    const int D = (int)x.size(-1);
    const int rows = (int)(x.numel() / D);
    b200::layernorm_fwd(bf16_ptr(x), bf16_ptr(gamma), bf16_ptr(beta), bf16_mut(y), f32_ptr(mean), f32_ptr(rstd), rows,
                        D, (float)eps, cur_stream());
}

void layernorm_bwd(Tensor dy, Tensor x, Tensor gamma, Tensor mean, Tensor rstd, OptT dres, Tensor dx, Tensor dgamma,
                   Tensor dbeta, OptT dxsum) {
    c10::cuda::CUDAGuard guard(x.device());
    const int D = (int)x.size(-1);
    const int rows = (int)(x.numel() / D);
    b200::layernorm_bwd(bf16_ptr(dy), bf16_ptr(x), bf16_ptr(gamma), f32_ptr(mean), f32_ptr(rstd),
                        dres.has_value() ? bf16_ptr(*dres) : nullptr, bf16_mut(dx), f32_ptr(dgamma), f32_ptr(dbeta),
                        dxsum.has_value() ? f32_ptr(*dxsum) : nullptr, rows, D, cur_stream());
}

void softmax_fwd(Tensor s, int64_t rows, int64_t n, int64_t ld, double scale) {
    c10::cuda::CUDAGuard guard(s.device());
    b200::softmax_fwd(bf16_mut(s), rows, (int)n, ld, (float)scale, cur_stream());
}
void softmax_bwd(Tensor dp, Tensor p, int64_t rows, int64_t n, int64_t ld, double scale) {
    c10::cuda::CUDAGuard guard(p.device());
    b200::softmax_bwd(bf16_mut(dp), bf16_ptr(p), rows, (int)n, ld, (float)scale, cur_stream());
}

bool attention_supported(int64_t N, int64_t hd) { return b200::attention_supported((int)N, (int)hd); }

// Argument checks of the attention entry points, all made before anything is launched.  The kernels read q / k / v
// and dO through TMA (16-byte aligned base, row stride a multiple of 8 elements), read O as bf16 pairs in the delta
// kernel, store O, dqkv and the probabilities as bf16 pairs (4-byte aligned, even row stride) and read lse / delta as
// float2 in the dK / dV role (8-byte aligned).
inline bool aligned(const Tensor& t, int64_t bytes) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % bytes == 0; }

// A [rows, cols] bf16 matrix with unit column stride on qkv's device, row stride >= cols and a multiple of ld_mult,
// base aligned to `align` bytes.
void check_matrix(const char* what, const char* name, const Tensor& t, const Tensor& like, int64_t rows, int64_t cols,
                  int64_t ld_mult, int64_t align) {
    TORCH_CHECK(t.is_cuda() && t.device() == like.device() && t.scalar_type() == at::kBFloat16, what, ": ", name,
                " must be a bf16 tensor on ", like.device());
    TORCH_CHECK(t.dim() == 2 && t.size(0) == rows && t.size(1) == cols, what, ": ", name, " must be [", rows, ", ",
                cols, "], got ", t.sizes());
    TORCH_CHECK(t.stride(1) == 1 && t.stride(0) >= cols && t.stride(0) % ld_mult == 0, what, ": ", name,
                " needs unit column stride and a row stride >= ", cols, " that is a multiple of ", ld_mult, ", got ",
                t.strides());
    TORCH_CHECK(aligned(t, align), what, ": ", name, " must be ", align, "-byte aligned");
}

// A contiguous fp32 vector of n elements on qkv's device, base aligned to `align` bytes.
void check_f32(const char* what, const char* name, const Tensor& t, const Tensor& like, int64_t n, int64_t align) {
    TORCH_CHECK(t.is_cuda() && t.device() == like.device() && t.scalar_type() == at::kFloat, what, ": ", name,
                " must be an fp32 tensor on ", like.device());
    TORCH_CHECK(t.is_contiguous() && t.numel() == n, what, ": ", name, " must be contiguous with ", n,
                " elements, got ", t.sizes());
    TORCH_CHECK(aligned(t, align), what, ": ", name, " must be ", align, "-byte aligned");
}

void check_attention_dims(const char* what, int64_t B, int64_t N, int64_t H, int64_t hd, double drop_p) {
    TORCH_CHECK(B >= 1 && H >= 1, what, ": need B >= 1 and H >= 1");
    TORCH_CHECK(b200::attention_shape_ok((int)N, (int)hd), what, ": unsupported (N, head_dim) = (", N, ", ", hd, ")");
    TORCH_CHECK(drop_p == 0.0 || (drop_p > 0.0 && drop_p < 1.0), what, ": dropout p must be 0 or in (0, 1)");
}

// drop_p > 0: attention dropout with the mask `dropout` draws for drop_key over [B*H, N, pad8(N)] probabilities.
void attention_fwd(Tensor qkv, Tensor out, OptT lse, OptT probs, int64_t B, int64_t N, int64_t H, int64_t hd,
                   double drop_p, int64_t drop_key) {
    c10::cuda::CUDAGuard guard(qkv.device());
    const char* what = "attention_fwd";
    check_attention_dims(what, B, N, H, hd, drop_p);
    const int64_t D = H * hd;
    check_matrix(what, "qkv", qkv, qkv, B * N, 3 * D, 8, 16);
    check_matrix(what, "out", out, qkv, B * N, D, 2, 4);
    TORCH_CHECK(out.is_contiguous(), "attention_fwd: out must be contiguous (the kernels store it with row stride D)");
    if (lse.has_value()) check_f32(what, "lse", *lse, qkv, B * H * N, 4);
    TORCH_CHECK(drop_p == 0.0 || !probs.has_value(), "attention_fwd: no probability output with dropout");
    if (probs.has_value()) {
        const Tensor& p = *probs;
        TORCH_CHECK(p.is_cuda() && p.device() == qkv.device() && p.scalar_type() == at::kBFloat16,
                    "attention_fwd: probs must be a bf16 tensor on ", qkv.device());
        TORCH_CHECK(p.dim() == 3 && p.size(0) == B * H && p.size(1) == N && p.size(2) >= N && p.size(2) % 2 == 0,
                    "attention_fwd: probs must be [B*H, N, ldp] with an even ldp >= N, got ", p.sizes());
        TORCH_CHECK(p.is_contiguous() && aligned(p, 4), "attention_fwd: probs must be contiguous and 4-byte aligned");
    }
    b200::attention_fwd(bf16_ptr(qkv), qkv.stride(0), bf16_mut(out), lse.has_value() ? f32_ptr(*lse) : nullptr,
                        probs.has_value() ? bf16_mut(*probs) : nullptr, probs.has_value() ? probs->size(2) : 0, (int)B,
                        (int)N, (int)H, (int)hd, cur_stream(), (float)drop_p, (uint64_t)drop_key);
}

void attention_bwd(Tensor qkv, Tensor dout, Tensor out, Tensor lse, Tensor delta, Tensor dqkv, OptT colsum, int64_t B,
                   int64_t N, int64_t H, int64_t hd, double drop_p, int64_t drop_key) {
    c10::cuda::CUDAGuard guard(qkv.device());
    const char* what = "attention_bwd";
    check_attention_dims(what, B, N, H, hd, drop_p);
    const int64_t D = H * hd;
    check_matrix(what, "qkv", qkv, qkv, B * N, 3 * D, 8, 16);
    check_matrix(what, "dout", dout, qkv, B * N, D, 8, 16);
    check_matrix(what, "out", out, qkv, B * N, D, 2, 4);
    check_f32(what, "lse", lse, qkv, B * H * N, 8);
    check_f32(what, "delta", delta, qkv, B * H * N, 8);
    check_matrix(what, "dqkv", dqkv, qkv, B * N, 3 * D, 2, 4);
    TORCH_CHECK(dqkv.is_contiguous(), "attention_bwd: dqkv must be contiguous (the kernels store it with row stride 3 D)");
    if (colsum.has_value()) check_f32(what, "colsum", *colsum, qkv, 3 * D, 4);
    b200::attention_bwd(bf16_ptr(qkv), qkv.stride(0), bf16_ptr(dout), dout.stride(0), bf16_ptr(out), out.stride(0),
                        f32_ptr(lse), f32_ptr(delta), bf16_mut(dqkv), (int)B, (int)N, (int)H, (int)hd, cur_stream(),
                        colsum.has_value() ? f32_ptr(*colsum) : nullptr, (float)drop_p, (uint64_t)drop_key);
}

// lam < 1: mixed targets (row b with row B-1-b); smoothing > 0: label smoothing.  The defaults are the hard loss.
void cross_entropy(Tensor logits, Tensor target, OptT dlogits, Tensor loss, OptT correct, double lam,
                   double smoothing) {
    c10::cuda::CUDAGuard guard(logits.device());
    TORCH_CHECK(target.scalar_type() == at::kLong && target.is_cuda(), "target must be a CUDA int64 tensor");
    TORCH_CHECK(lam >= 0.0 && lam <= 1.0 && smoothing >= 0.0 && smoothing < 1.0,
                "cross_entropy: lam must be in [0, 1] and smoothing in [0, 1)");
    const int B = (int)logits.size(0), C = (int)logits.size(1);
    b200::cross_entropy(bf16_ptr(logits), reinterpret_cast<const int64_t*>(target.data_ptr()),
                        dlogits.has_value() ? bf16_mut(*dlogits) : nullptr, f32_ptr(loss),
                        correct.has_value() ? reinterpret_cast<int*>(correct->data_ptr()) : nullptr, B, C,
                        cur_stream(), lam, smoothing);
}

// lam given: mix image b with image B-1-b, Mixup with an empty box, CutMix with box = [yl, yh, xl, xh].
void im2col(Tensor img, Tensor cols, int64_t P, std::optional<double> lam, std::vector<int64_t> box) {
    c10::cuda::CUDAGuard guard(img.device());
    TORCH_CHECK(img.is_contiguous() && img.dim() == 4 && img.size(1) == 3, "images must be contiguous [B,3,S,S]");
    const bool is_bf16 = img.scalar_type() == at::kBFloat16;
    TORCH_CHECK(is_bf16 || img.scalar_type() == at::kFloat, "images must be fp32 or bf16");
    b200::Im2colMix mix;
    if (lam.has_value()) {
        TORCH_CHECK(*lam >= 0.0 && *lam <= 1.0, "im2col: lam must be in [0, 1]");
        TORCH_CHECK(box.empty() || box.size() == 4, "im2col: box must be [] or [yl, yh, xl, xh]");
        mix.lam = (float)*lam, mix.mlam = (float)(1.0 - *lam);
        mix.mode = box.empty() ? 1 : 2;
        if (!box.empty()) mix.yl = (int)box[0], mix.yh = (int)box[1], mix.xl = (int)box[2], mix.xh = (int)box[3];
    } else {
        TORCH_CHECK(box.empty(), "im2col: a CutMix box needs lam");
    }
    b200::im2col(img.data_ptr(), is_bf16, bf16_mut(cols), (int)img.size(0), (int)img.size(2), (int)P,
                 (int)cols.size(1), cur_stream(), mix);
}

void gelu_fwd(Tensor u, Tensor g) {
    c10::cuda::CUDAGuard guard(u.device());
    b200::gelu_fwd(bf16_ptr(u), bf16_mut(g), u.numel(), cur_stream());
}
void dropout(Tensor x, Tensor y, double p, int64_t key) {
    c10::cuda::CUDAGuard guard(x.device());
    TORCH_CHECK(x.is_contiguous() && y.is_contiguous() && x.numel() == y.numel(), "dropout: contiguous, same size");
    b200::dropout(bf16_ptr(x), bf16_mut(y), x.numel(), (float)p, (uint64_t)key, cur_stream());
}
void drop_path_scale(Tensor scale, int64_t sample_offset, double p, int64_t key) {
    c10::cuda::CUDAGuard guard(scale.device());
    TORCH_CHECK(scale.is_contiguous() && scale.dim() == 1, "drop_path_scale: contiguous [B] fp32 output");
    b200::drop_path_scale(f32_ptr(scale), (int)scale.numel(), sample_offset, (float)p, (uint64_t)key, cur_stream());
}
void drop_path_bwd(Tensor dy, Tensor scale, Tensor dt, Tensor colsum, int64_t N) {
    c10::cuda::CUDAGuard guard(dy.device());
    TORCH_CHECK(dy.dim() == 2 && dy.is_contiguous() && dt.is_contiguous() && dt.sizes() == dy.sizes(),
                "drop_path_bwd: contiguous [T, C] dy and dt");
    TORCH_CHECK(scale.is_contiguous() && scale.numel() * N == dy.size(0), "drop_path_bwd: one scale per N rows");
    TORCH_CHECK(colsum.is_contiguous() && colsum.numel() == dy.size(1), "drop_path_bwd: colsum must be [C]");
    b200::drop_path_bwd(bf16_ptr(dy), f32_ptr(scale), bf16_mut(dt), f32_ptr(colsum), dy.size(0), (int)dy.size(1),
                        (int)N, cur_stream());
}
void meanpool_fwd(Tensor xn, Tensor pooled, int64_t B, int64_t N) {
    c10::cuda::CUDAGuard guard(xn.device());
    TORCH_CHECK(xn.is_contiguous() && pooled.is_contiguous() && xn.numel() == pooled.numel() * N, "meanpool: bad shapes");
    b200::meanpool_fwd(bf16_ptr(xn), bf16_mut(pooled), (int)B, (int)N, (int)(pooled.numel() / B), cur_stream());
}
void meanpool_bwd(Tensor dpooled, Tensor dxn, int64_t B, int64_t N) {
    c10::cuda::CUDAGuard guard(dxn.device());
    TORCH_CHECK(dxn.is_contiguous() && dpooled.is_contiguous() && dxn.numel() == dpooled.numel() * N, "meanpool: bad shapes");
    b200::meanpool_bwd(bf16_ptr(dpooled), bf16_mut(dxn), (int)B, (int)N, (int)(dpooled.numel() / B), cur_stream());
}
void dgelu_mul(Tensor dg, Tensor u, Tensor du) {
    c10::cuda::CUDAGuard guard(u.device());
    b200::dgelu_mul(bf16_ptr(dg), bf16_ptr(u), bf16_mut(du), u.numel(), cur_stream());
}
// u [M, Hd] packed [gate | value]; g [M, Hd / 2]; dg [M, Hd / 2]; du [M, Hd]; all contiguous.
void swiglu_fwd(Tensor u, Tensor g) {
    c10::cuda::CUDAGuard guard(u.device());
    TORCH_CHECK(u.dim() == 2 && g.dim() == 2 && u.is_contiguous() && g.is_contiguous(),
                "swiglu_fwd: contiguous 2-D u and g");
    TORCH_CHECK(g.size(0) == u.size(0) && 2 * g.size(1) == u.size(1), "swiglu_fwd: g must be [M, Hd / 2] for u [M, Hd]");
    b200::swiglu_fwd(bf16_ptr(u), bf16_mut(g), u.size(0), u.size(1), cur_stream());
}
void swiglu_bwd(Tensor dg, Tensor u, Tensor du) {
    c10::cuda::CUDAGuard guard(u.device());
    TORCH_CHECK(u.dim() == 2 && dg.dim() == 2 && du.dim() == 2 && u.is_contiguous() && dg.is_contiguous() &&
                    du.is_contiguous(), "swiglu_bwd: contiguous 2-D dg, u and du");
    TORCH_CHECK(dg.size(0) == u.size(0) && 2 * dg.size(1) == u.size(1) && du.sizes() == u.sizes(),
                "swiglu_bwd: dg must be [M, Hd / 2] and du [M, Hd] for u [M, Hd]");
    b200::swiglu_bwd(bf16_ptr(dg), bf16_ptr(u), bf16_mut(du), u.size(0), u.size(1), cur_stream());
}

// qkv / out: [T, >= 3 H hd] row-major bf16 (out may be qkv: in place); mean / rstd: fp32 [T * 2 * H].
void qk_norm_fwd(Tensor qkv, Tensor wq, Tensor bq, Tensor wk, Tensor bk, Tensor out, Tensor mean, Tensor rstd,
                 int64_t H, int64_t hd, double eps) {
    c10::cuda::CUDAGuard guard(qkv.device());
    TORCH_CHECK(qkv.dim() == 2 && qkv.stride(1) == 1 && out.dim() == 2 && out.stride(1) == 1 &&
                    out.size(0) == qkv.size(0), "qk_norm_fwd: qkv and out must be row-major [T, 3D] matrices");
    const int64_t T = qkv.size(0);
    for (const Tensor* w : {&wq, &bq, &wk, &bk})
        TORCH_CHECK(w->is_contiguous() && w->numel() == hd, "qk_norm_fwd: weights and biases must be contiguous [hd]");
    TORCH_CHECK(mean.is_contiguous() && rstd.is_contiguous() && mean.numel() == T * 2 * H && rstd.numel() == T * 2 * H,
                "qk_norm_fwd: mean / rstd must be contiguous [T * 2 * H]");
    b200::qk_norm_fwd(bf16_ptr(qkv), qkv.stride(0), bf16_ptr(wq), bf16_ptr(bq), bf16_ptr(wk), bf16_ptr(bk),
                      bf16_mut(out), out.stride(0), f32_ptr(mean), f32_ptr(rstd), (int)T, (int)H, (int)hd, (float)eps,
                      cur_stream());
}
void qk_norm_bwd(Tensor dqkv, Tensor qkv, Tensor wq, Tensor wk, Tensor mean, Tensor rstd, Tensor dwq, Tensor dbq,
                 Tensor dwk, Tensor dbk, Tensor colsum, int64_t H, int64_t hd) {
    c10::cuda::CUDAGuard guard(qkv.device());
    TORCH_CHECK(qkv.dim() == 2 && qkv.stride(1) == 1 && dqkv.dim() == 2 && dqkv.stride(1) == 1 &&
                    dqkv.size(0) == qkv.size(0), "qk_norm_bwd: qkv and dqkv must be row-major [T, 3D] matrices");
    const int64_t T = qkv.size(0);
    TORCH_CHECK(wq.is_contiguous() && wk.is_contiguous() && wq.numel() == hd && wk.numel() == hd,
                "qk_norm_bwd: weights must be contiguous [hd]");
    TORCH_CHECK(mean.is_contiguous() && rstd.is_contiguous() && mean.numel() == T * 2 * H && rstd.numel() == T * 2 * H,
                "qk_norm_bwd: mean / rstd must be contiguous [T * 2 * H]");
    for (const Tensor* a : {&dwq, &dbq, &dwk, &dbk})
        TORCH_CHECK(a->is_contiguous() && a->numel() == hd, "qk_norm_bwd: dw / db must be contiguous fp32 [hd]");
    TORCH_CHECK(colsum.is_contiguous() && colsum.numel() >= 2 * H * hd, "qk_norm_bwd: colsum must be fp32 [>= 2 H hd]");
    b200::qk_norm_bwd(bf16_mut(dqkv), dqkv.stride(0), bf16_ptr(qkv), qkv.stride(0), bf16_ptr(wq), bf16_ptr(wk),
                      f32_ptr(mean), f32_ptr(rstd), f32_ptr(dwq), f32_ptr(dbq), f32_ptr(dwk), f32_ptr(dbk),
                      f32_ptr(colsum), (int)T, (int)H, (int)hd, cur_stream());
}

// LayerScale folded into a linear layer.  W / dW / Wg: contiguous bf16 [D, K]; b / gamma / bg: contiguous bf16 [D];
// S / db / dgamma: contiguous fp32 [D].
void check_layer_scale(const char* what, const Tensor& W, const Tensor& b, const Tensor& gamma, const Tensor& Wg) {
    TORCH_CHECK(W.is_cuda() && W.scalar_type() == at::kBFloat16 && W.dim() == 2 && W.is_contiguous(), what,
                ": W must be a contiguous bf16 CUDA [D, K] matrix");
    TORCH_CHECK(Wg.scalar_type() == at::kBFloat16 && Wg.is_contiguous() && Wg.sizes() == W.sizes(), what,
                ": Wg must be a contiguous bf16 matrix of W's shape");
    for (const Tensor* t : {&b, &gamma})
        TORCH_CHECK(t->scalar_type() == at::kBFloat16 && t->is_contiguous() && t->numel() == W.size(0), what,
                    ": b and gamma must be contiguous bf16 vectors of length D = W.size(0)");
}
void layer_scale_fold(Tensor W, Tensor b, Tensor gamma, Tensor Wg, Tensor bg) {
    c10::cuda::CUDAGuard guard(W.device());
    check_layer_scale("layer_scale_fold", W, b, gamma, Wg);
    TORCH_CHECK(bg.scalar_type() == at::kBFloat16 && bg.is_contiguous() && bg.numel() == W.size(0),
                "layer_scale_fold: bg must be a contiguous bf16 vector of length D = W.size(0)");
    b200::layer_scale_fold(bf16_ptr(W), bf16_ptr(b), bf16_ptr(gamma), bf16_mut(Wg), bf16_mut(bg), W.size(0), W.size(1),
                           cur_stream());
}
void layer_scale_bwd(Tensor W, Tensor b, Tensor gamma, Tensor dW, Tensor S, Tensor Wg, Tensor db, Tensor dgamma) {
    c10::cuda::CUDAGuard guard(W.device());
    check_layer_scale("layer_scale_bwd", W, b, gamma, Wg);
    TORCH_CHECK(dW.scalar_type() == at::kBFloat16 && dW.is_contiguous() && dW.sizes() == W.sizes(),
                "layer_scale_bwd: dW must be a contiguous bf16 matrix of W's shape");
    for (const Tensor* t : {&S, &db, &dgamma})
        TORCH_CHECK(t->scalar_type() == at::kFloat && t->is_contiguous() && t->numel() == W.size(0),
                    "layer_scale_bwd: S, db and dgamma must be contiguous fp32 vectors of length D = W.size(0)");
    b200::layer_scale_bwd(bf16_ptr(W), bf16_ptr(b), bf16_ptr(gamma), bf16_mut(dW), f32_ptr(S), bf16_mut(Wg),
                          f32_ptr(db), f32_ptr(dgamma), W.size(0), W.size(1), cur_stream());
}

// Prefix tokens (class + register tokens).  y: contiguous bf16 [B * N, D] patch rows; cls: bf16 [D]; reg: bf16
// [R, D] or None (R = 0); pos: bf16 [P, D] (P = 1 + R) or None; x0: contiguous bf16 [B * (N + P), D].
void check_bf16_buf(const char* what, const char* name, const Tensor& t, int64_t numel) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16, what, ": ", name, " must be a bf16 CUDA tensor");
    TORCH_CHECK(t.is_contiguous() && t.numel() == numel, what, ": ", name, " must be contiguous with ", numel,
                " elements, got ", t.numel());
}
void tokens_fwd(Tensor y, Tensor cls, OptT reg, OptT pos, Tensor x0, int64_t B, int64_t N) {
    c10::cuda::CUDAGuard guard(y.device());
    TORCH_CHECK(y.dim() == 2, "tokens_fwd: y must be a [B * N, D] matrix");
    const int64_t D = y.size(1);
    TORCH_CHECK(D % 8 == 0, "tokens_fwd: need D % 8 == 0 (16-byte vectors), got D ", D);
    check_bf16_buf("tokens_fwd", "y", y, B * N * D);
    check_bf16_buf("tokens_fwd", "cls", cls, D);
    int64_t P = 1;
    if (reg.has_value()) {
        TORCH_CHECK(reg->numel() % D == 0 && reg->numel() > 0, "tokens_fwd: reg must be [R, D] with R >= 1");
        P += reg->numel() / D;
        check_bf16_buf("tokens_fwd", "reg", *reg, (P - 1) * D);
    }
    if (pos.has_value()) check_bf16_buf("tokens_fwd", "pos", *pos, P * D);
    check_bf16_buf("tokens_fwd", "x0", x0, B * (N + P) * D);
    b200::tokens_fwd(bf16_ptr(y), bf16_ptr(cls), reg.has_value() ? bf16_ptr(*reg) : nullptr,
                     pos.has_value() ? bf16_ptr(*pos) : nullptr, bf16_mut(x0), B, N, P, D, cur_stream());
}
// dx0: contiguous bf16 [B * (N + P), D]; dpatch: contiguous bf16 [B * N, D]; dtok: contiguous fp32 [N + P, D].
void tokens_bwd(Tensor dx0, Tensor dpatch, Tensor dtok, int64_t B, int64_t N, int64_t P) {
    c10::cuda::CUDAGuard guard(dx0.device());
    TORCH_CHECK(P >= 1, "tokens_bwd: need P >= 1 prefix tokens, got P ", P);
    TORCH_CHECK(dx0.dim() == 2, "tokens_bwd: dx0 must be a [B * (N + P), D] matrix");
    const int64_t D = dx0.size(1);
    TORCH_CHECK(D % 8 == 0, "tokens_bwd: need D % 8 == 0 (16-byte vectors), got D ", D);
    check_bf16_buf("tokens_bwd", "dx0", dx0, B * (N + P) * D);
    check_bf16_buf("tokens_bwd", "dpatch", dpatch, B * N * D);
    TORCH_CHECK(dtok.is_cuda() && dtok.scalar_type() == at::kFloat && dtok.is_contiguous() &&
                    dtok.numel() == (N + P) * D,
                "tokens_bwd: dtok must be a contiguous fp32 CUDA tensor with (N + P) * D elements");
    b200::tokens_bwd(bf16_ptr(dx0), bf16_mut(dpatch), f32_ptr(dtok), B, N, P, D, cur_stream());
}

// Patch dropout.  keep: contiguous int32 [B, K]; inv: contiguous int32 [B, N].
void check_i32(const char* what, const char* name, const Tensor& t, int64_t rows, int64_t cols) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kInt && t.is_contiguous() && t.dim() == 2 && t.size(0) == rows &&
                    t.size(1) == cols,
                what, ": ", name, " must be a contiguous int32 CUDA tensor [", rows, ", ", cols, "]");
}
void patch_drop_select(Tensor keep, Tensor inv, int64_t N, int64_t K, int64_t offset, int64_t key) {
    c10::cuda::CUDAGuard guard(keep.device());
    const int64_t B = keep.dim() == 2 ? keep.size(0) : 0;
    check_i32("patch_drop_select", "keep", keep, B, K);
    check_i32("patch_drop_select", "inv", inv, B, N);
    b200::patch_drop_select(keep.data_ptr<int>(), inv.data_ptr<int>(), B, N, K, offset, (uint64_t)key, cur_stream());
}
// cols: [B * K, Kpad] bf16 for the kept patches keep [B, K]; lam / box as for im2col.
void im2col_gather(Tensor img, Tensor keep, Tensor cols, int64_t P, std::optional<double> lam,
                   std::vector<int64_t> box) {
    c10::cuda::CUDAGuard guard(img.device());
    TORCH_CHECK(img.is_contiguous() && img.dim() == 4 && img.size(1) == 3, "images must be contiguous [B,3,S,S]");
    const bool is_bf16 = img.scalar_type() == at::kBFloat16;
    TORCH_CHECK(is_bf16 || img.scalar_type() == at::kFloat, "images must be fp32 or bf16");
    TORCH_CHECK(keep.dim() == 2, "im2col_gather: keep must be [B, K]");
    const int64_t B = img.size(0), K = keep.size(1);
    check_i32("im2col_gather", "keep", keep, B, K);
    TORCH_CHECK(cols.is_contiguous() && cols.dim() == 2 && cols.size(0) == B * K,
                "im2col_gather: cols must be a contiguous [B * K, Kpad] matrix");
    b200::Im2colMix mix;
    if (lam.has_value()) {
        TORCH_CHECK(*lam >= 0.0 && *lam <= 1.0, "im2col_gather: lam must be in [0, 1]");
        TORCH_CHECK(box.empty() || box.size() == 4, "im2col_gather: box must be [] or [yl, yh, xl, xh]");
        mix.lam = (float)*lam, mix.mlam = (float)(1.0 - *lam);
        mix.mode = box.empty() ? 1 : 2;
        if (!box.empty()) mix.yl = (int)box[0], mix.yh = (int)box[1], mix.xl = (int)box[2], mix.xh = (int)box[3];
    } else {
        TORCH_CHECK(box.empty(), "im2col_gather: a CutMix box needs lam");
    }
    b200::im2col_gather(img.data_ptr(), is_bf16, keep.data_ptr<int>(), bf16_mut(cols), (int)B, (int)img.size(2),
                        (int)P, (int)cols.size(1), (int)K, cur_stream(), mix);
}
// pos: contiguous bf16 [N, D]; out: contiguous bf16 [B * K, D].
void pos_gather(Tensor pos, Tensor keep, Tensor out) {
    c10::cuda::CUDAGuard guard(pos.device());
    TORCH_CHECK(pos.dim() == 2 && keep.dim() == 2, "pos_gather: pos must be [N, D] and keep [B, K]");
    const int64_t N = pos.size(0), D = pos.size(1), B = keep.size(0), K = keep.size(1);
    TORCH_CHECK(K >= 1 && K <= N, "pos_gather: need 1 <= K <= N, got K ", K, ", N ", N);
    check_bf16_buf("pos_gather", "pos", pos, N * D);
    check_i32("pos_gather", "keep", keep, B, K);
    check_bf16_buf("pos_gather", "out", out, B * K * D);
    b200::pos_gather(bf16_ptr(pos), keep.data_ptr<int>(), bf16_mut(out), B * K, D, cur_stream());
}
// dx0: contiguous bf16 [B * (P + K), D]; inv: int32 [B, N]; dpatch: bf16 [B * K, D] or None; dtok: fp32 [P + N, D].
void patch_drop_bwd(Tensor dx0, Tensor inv, OptT dpatch, Tensor dtok, int64_t B, int64_t N, int64_t K, int64_t P) {
    c10::cuda::CUDAGuard guard(dx0.device());
    TORCH_CHECK(P >= 0, "patch_drop_bwd: need P >= 0 prefix tokens, got P ", P);
    TORCH_CHECK(K >= 1 && K <= N, "patch_drop_bwd: need 1 <= K <= N, got K ", K, ", N ", N);
    TORCH_CHECK(dx0.dim() == 2, "patch_drop_bwd: dx0 must be a [B * (P + K), D] matrix");
    const int64_t D = dx0.size(1);
    TORCH_CHECK(D % 8 == 0, "patch_drop_bwd: need D % 8 == 0 (16-byte vectors), got D ", D);
    check_bf16_buf("patch_drop_bwd", "dx0", dx0, B * (P + K) * D);
    check_i32("patch_drop_bwd", "inv", inv, B, N);
    if (dpatch.has_value()) check_bf16_buf("patch_drop_bwd", "dpatch", *dpatch, B * K * D);
    TORCH_CHECK(dtok.is_cuda() && dtok.scalar_type() == at::kFloat && dtok.is_contiguous() &&
                    dtok.numel() == (P + N) * D,
                "patch_drop_bwd: dtok must be a contiguous fp32 CUDA tensor with (P + N) * D elements");
    b200::patch_drop_bwd(bf16_ptr(dx0), inv.data_ptr<int>(), dpatch.has_value() ? bf16_mut(*dpatch) : nullptr,
                         f32_ptr(dtok), B, N, K, P, D, cur_stream());
}

void colsum(Tensor x, Tensor out) {
    c10::cuda::CUDAGuard guard(x.device());
    const int C = (int)x.size(-1);
    b200::colsum(bf16_ptr(x), f32_ptr(out), x.numel() / C, C, cur_stream());
}

void sumsq(Tensor x, Tensor out) {
    c10::cuda::CUDAGuard guard(x.device());
    const bool is_bf16 = x.scalar_type() == at::kBFloat16;
    TORCH_CHECK(is_bf16 || x.scalar_type() == at::kFloat, "sumsq: fp32 or bf16 only");
    b200::sumsq(x.data_ptr(), is_bf16, x.numel(), f32_ptr(out), cur_stream());
}

// Parameter groups of the grouped AdamW kernels: `groups` uint8 [n / 64] (the group of every 64-element chunk),
// `group_hyper` fp32 [G, 2] rows of (lr_scale, wd); both or neither.  Returns false when neither is given.
bool check_groups(const char* who, const OptT& groups, const OptT& group_hyper, int64_t n, const at::Device& dev) {
    TORCH_CHECK(groups.has_value() == group_hyper.has_value(), who, ": pass both groups and group_hyper, or neither");
    if (!groups.has_value()) return false;
    TORCH_CHECK(groups->scalar_type() == at::kByte && group_hyper->scalar_type() == at::kFloat, who,
                ": groups must be uint8 and group_hyper fp32");
    TORCH_CHECK(groups->device() == dev && group_hyper->device() == dev && groups->is_contiguous() &&
                    group_hyper->is_contiguous(), who, ": groups and group_hyper must be contiguous, on the shard's device");
    TORCH_CHECK(n % 64 == 0 && groups->numel() == n / 64, who, ": ", n, " elements need n % 64 == 0 and n / 64 chunk "
                "groups, got ", groups->numel());
    TORCH_CHECK(group_hyper->dim() == 2 && group_hyper->size(1) == 2 && group_hyper->size(0) >= 1 &&
                    group_hyper->size(0) <= 256, who, ": group_hyper must be [G, 2] with 1 <= G <= 256");
    return true;
}

void adamw_split(Tensor hi, Tensor lo, Tensor m, Tensor v, Tensor grad, OptT clip_coef, double lr, double beta1,
                 double beta2, double eps, double wd, int64_t step, OptT hyper, OptT ema_hi, OptT ema_lo,
                 double ema_decay, OptT groups, OptT group_hyper) {
    c10::cuda::CUDAGuard guard(hi.device());
    const bool grouped = check_groups("adamw_split", groups, group_hyper, hi.numel(), hi.device());
    TORCH_CHECK(hi.scalar_type() == at::kBFloat16 && lo.scalar_type() == at::kShort, "hi: bf16, lo: int16");
    TORCH_CHECK(ema_hi.has_value() == ema_lo.has_value(), "adamw_split: pass both ema_hi and ema_lo, or neither");
    if (ema_hi.has_value()) {
        TORCH_CHECK(ema_hi->scalar_type() == at::kBFloat16 && ema_lo->scalar_type() == at::kShort,
                    "adamw_split: ema_hi must be bf16 and ema_lo int16");
        TORCH_CHECK(ema_hi->numel() == hi.numel() && ema_lo->numel() == hi.numel(),
                    "adamw_split: the EMA must have as many elements as the master");
        TORCH_CHECK(ema_hi->is_contiguous() && ema_lo->is_contiguous() && ema_hi->device() == hi.device() &&
                        ema_lo->device() == hi.device(), "adamw_split: the EMA must be contiguous, on the master's device");
        TORCH_CHECK(ema_decay >= 0.0 && ema_decay < 1.0, "adamw_split: ema_decay must be in [0, 1)");
    }
    const bool gbf = grad.scalar_type() == at::kBFloat16;
    b200::adamw_split(reinterpret_cast<uint16_t*>(hi.data_ptr()), reinterpret_cast<int16_t*>(lo.data_ptr()),
                      f32_ptr(m), f32_ptr(v), grad.data_ptr(), gbf, hi.numel(),
                      clip_coef.has_value() ? f32_ptr(*clip_coef) : nullptr, (float)lr, (float)beta1, (float)beta2,
                      (float)eps, (float)wd, (int)step, cur_stream(), hyper.has_value() ? f32_ptr(*hyper) : nullptr,
                      ema_hi.has_value() ? reinterpret_cast<uint16_t*>(ema_hi->data_ptr()) : nullptr,
                      ema_lo.has_value() ? reinterpret_cast<int16_t*>(ema_lo->data_ptr()) : nullptr, (float)ema_decay,
                      grouped ? groups->data_ptr<uint8_t>() : nullptr, grouped ? f32_ptr(*group_hyper) : nullptr);
}

void adamw_fp32(Tensor w, Tensor m, Tensor v, Tensor grad, OptT clip_coef, double lr, double beta1, double beta2,
                double eps, double wd, int64_t step, OptT ema, double ema_decay, OptT groups, OptT group_hyper) {
    c10::cuda::CUDAGuard guard(w.device());
    const bool grouped = check_groups("adamw_fp32", groups, group_hyper, w.numel(), w.device());
    if (ema.has_value()) {
        TORCH_CHECK(ema->scalar_type() == at::kFloat && ema->numel() == w.numel() && ema->is_contiguous() &&
                        ema->device() == w.device(), "adamw_fp32: the EMA must be a contiguous fp32 tensor like w");
        TORCH_CHECK(ema_decay >= 0.0 && ema_decay < 1.0, "adamw_fp32: ema_decay must be in [0, 1)");
    }
    const bool gbf = grad.scalar_type() == at::kBFloat16;
    b200::adamw_fp32(f32_ptr(w), f32_ptr(m), f32_ptr(v), grad.data_ptr(), gbf, w.numel(),
                     clip_coef.has_value() ? f32_ptr(*clip_coef) : nullptr, (float)lr, (float)beta1, (float)beta2,
                     (float)eps, (float)wd, (int)step, cur_stream(), ema.has_value() ? f32_ptr(*ema) : nullptr,
                     (float)ema_decay, grouped ? groups->data_ptr<uint8_t>() : nullptr,
                     grouped ? f32_ptr(*group_hyper) : nullptr);
}

void split_fp32(Tensor w, Tensor hi, Tensor lo) {
    c10::cuda::CUDAGuard guard(w.device());
    b200::split_fp32(f32_ptr(w), reinterpret_cast<uint16_t*>(hi.data_ptr()), reinterpret_cast<int16_t*>(lo.data_ptr()),
                     w.numel(), cur_stream());
}
void merge_fp32(Tensor hi, Tensor lo, Tensor w) {
    c10::cuda::CUDAGuard guard(w.device());
    b200::merge_fp32(reinterpret_cast<const uint16_t*>(hi.data_ptr()), reinterpret_cast<const int16_t*>(lo.data_ptr()),
                     f32_ptr(w), w.numel(), cur_stream());
}
void clip_coef(Tensor sumsq_in, double max_norm, Tensor coef, OptT norm_out) {
    c10::cuda::CUDAGuard guard(coef.device());
    b200::clip_coef(f32_ptr(sumsq_in), (float)max_norm, f32_ptr(coef),
                    norm_out.has_value() ? f32_ptr(*norm_out) : nullptr, cur_stream());
}

// ---- NVLink / NVSwitch collectives over symmetric memory (raw device pointers from torch symm_mem) ----
inline const int64_t* seg_ptr(const Tensor& t) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kLong && t.is_contiguous(), "segment table: CUDA int64");
    return reinterpret_cast<const int64_t*>(t.data_ptr());
}
void p2p_all_gather(std::vector<int64_t> peer_ptrs, int64_t rank, Tensor out, Tensor seg_table, int64_t total_chunks,
                    int64_t max_ctas) {
    c10::cuda::CUDAGuard guard(out.device());
    b200::p2p_all_gather(peer_ptrs, (int)rank, out.data_ptr(), seg_ptr(seg_table), (int)seg_table.size(0),
                         total_chunks, (int)max_ctas, cur_stream());
}
// Copy-engine transport of the all-gather: one asynchronous device-to-device copy per (parameter group, source rank)
// straight from the peer's symmetric shard into its final place in the gathered buffer.  No SM, no shared memory, no
// registers are taken from the GEMM running next to it.  Graph-capturable (memcpy nodes).  Its rate against the pull
// kernel has not been measured on H100.
void ce_all_gather(std::vector<int64_t> src_ptrs, std::vector<int64_t> dst_ptrs, std::vector<int64_t> nbytes) {
    TORCH_CHECK(src_ptrs.size() == dst_ptrs.size() && src_ptrs.size() == nbytes.size(), "ce_all_gather: ragged lists");
    cudaStream_t stream = cur_stream();
    for (size_t i = 0; i < src_ptrs.size(); ++i) {
        cudaError_t err = cudaMemcpyAsync(reinterpret_cast<void*>(dst_ptrs[i]), reinterpret_cast<const void*>(src_ptrs[i]),
                                          static_cast<size_t>(nbytes[i]), cudaMemcpyDeviceToDevice, stream);
        TORCH_CHECK(err == cudaSuccess, "ce_all_gather: ", cudaGetErrorString(err));
    }
}
// adam = [] or (hi, lo, m, v tensors given separately) + hyper = [lr, beta1, beta2, eps, wd, step]
bool make_adam(const OptT& hi, const OptT& lo, const OptT& m, const OptT& v, const std::vector<double>& hyper,
               b200::AdamFuse& a) {
    if (!hi.has_value()) return false;
    TORCH_CHECK(lo.has_value() && m.has_value() && v.has_value() && hyper.size() == 6, "bad fused-AdamW arguments");
    TORCH_CHECK(hi->scalar_type() == at::kBFloat16 && lo->scalar_type() == at::kShort, "hi: bf16, lo: int16");
    a.hi = reinterpret_cast<uint16_t*>(hi->data_ptr());
    a.lo = reinterpret_cast<int16_t*>(lo->data_ptr());
    a.m = f32_ptr(*m);
    a.v = f32_ptr(*v);
    a.lr = (float)hyper[0], a.beta1 = (float)hyper[1], a.beta2 = (float)hyper[2], a.eps = (float)hyper[3];
    a.wd = (float)hyper[4];
    // 1 - beta^t in double, as adamw_split does: in fp32, 1 - powf(0.999f, 2) keeps only the rounding error of powf
    // (several ulps of 0.002)
    const double step = hyper[5];
    a.inv_bc1 = 1.f / static_cast<float>(1.0 - std::pow(static_cast<double>(a.beta1), step));
    a.inv_bc2 = 1.f / static_cast<float>(1.0 - std::pow(static_cast<double>(a.beta2), step));
    return true;
}
inline uint32_t* seq_ptr(const OptT& t) {
    if (!t.has_value()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kInt, "sequence counters: CUDA int32 tensor");
    return reinterpret_cast<uint32_t*>(t->data_ptr());
}
// sync = [] (caller brackets with barriers) or [rank, world, slot_ready, slot_done, counter_idx] + flag_ptrs, seq_dev, cta_ctr
bool make_sync(const std::vector<int64_t>& sync, const std::vector<int64_t>& flag_ptrs, const OptT& seq_dev,
               const OptT& cta_ctr, b200::CommSync& cs) {
    if (sync.empty()) return false;
    TORCH_CHECK(sync.size() == 5 && seq_dev.has_value() && cta_ctr.has_value(), "bad collective sync arguments");
    cs.flag_ptrs = flag_ptrs;
    cs.rank = (int)sync[0], cs.world = (int)sync[1], cs.slot_ready = (int)sync[2], cs.slot_done = (int)sync[3];
    cs.counter_idx = (int)sync[4];
    cs.seq_dev = seq_ptr(seq_dev);
    cs.cta_ctr = seq_ptr(cta_ctr);
    return true;
}
void reduce_scatter(std::vector<int64_t> peer_ptrs, int64_t mc_ptr, int64_t rank, int64_t world, Tensor out,
                    Tensor seg_table, int64_t total_chunks, bool in_is_bf16, double scale, OptT sumsq_out,
                    int64_t max_ctas, std::vector<int64_t> sync, std::vector<int64_t> flag_ptrs, OptT seq_dev,
                    OptT cta_ctr, OptT hi, OptT lo, OptT m, OptT v, std::vector<double> hyper, OptT groups,
                    OptT group_hyper) {
    c10::cuda::CUDAGuard guard(out.device());
    b200::AdamFuse a;
    const bool fused = make_adam(hi, lo, m, v, hyper, a);
    TORCH_CHECK(fused || !groups.has_value(), "reduce_scatter: parameter groups need the fused-AdamW arguments");
    if (fused && check_groups("reduce_scatter", groups, group_hyper, hi->numel(), hi->device())) {
        a.groups = groups->data_ptr<uint8_t>();
        a.group_hyper = f32_ptr(*group_hyper);
    }
    b200::CommSync cs;
    const bool synced = make_sync(sync, flag_ptrs, seq_dev, cta_ctr, cs);
    b200::reduce_scatter(peer_ptrs, mc_ptr, (int)rank, (int)world, f32_ptr(out), seg_ptr(seg_table),
                         (int)seg_table.size(0), total_chunks, in_is_bf16, (float)scale,
                         sumsq_out.has_value() ? f32_ptr(*sumsq_out) : nullptr, (int)max_ctas, cur_stream(),
                         synced ? &cs : nullptr, fused ? &a : nullptr);
}
void all_reduce_mean(std::vector<int64_t> peer_ptrs, int64_t mc_ptr, int64_t rank, int64_t world, Tensor buf,
                     int64_t max_ctas, std::vector<int64_t> sync, std::vector<int64_t> flag_ptrs, OptT seq_dev,
                     OptT cta_ctr) {
    c10::cuda::CUDAGuard guard(buf.device());
    TORCH_CHECK(buf.scalar_type() == at::kBFloat16 && buf.is_contiguous(), "all_reduce_mean: contiguous bf16 buffer");
    b200::CommSync cs;
    TORCH_CHECK(make_sync(sync, flag_ptrs, seq_dev, cta_ctr, cs), "all_reduce_mean needs the flag protocol");
    b200::all_reduce_mean_bf16(peer_ptrs, mc_ptr, (int)rank, (int)world, buf.numel() * 2, 1.0f / (float)world,
                               (int)max_ctas, cur_stream(), &cs);
}
void signal_barrier(std::vector<int64_t> flag_ptrs, int64_t rank, int64_t world, int64_t slot, int64_t seq,
                    OptT seq_dev) {
    b200::signal_barrier(flag_ptrs, (int)rank, (int)world, (int)slot, (uint32_t)seq, cur_stream(), seq_ptr(seq_dev));
}
void allreduce_scalars(std::vector<int64_t> flag_ptrs, std::vector<int64_t> scratch_ptrs, int64_t rank, int64_t world,
                       int64_t slot, int64_t seq, Tensor vals, int64_t op, OptT seq_dev, int64_t counter_idx) {
    c10::cuda::CUDAGuard guard(vals.device());
    b200::allreduce_scalars(flag_ptrs, scratch_ptrs, (int)rank, (int)world, (int)slot, (uint32_t)seq, f32_ptr(vals),
                            (int)vals.numel(), (int)op, cur_stream(), seq_ptr(seq_dev), (int)counter_idx);
}
int64_t ag_chunk_bytes() { return b200::ag_chunk_bytes(); }
int64_t rs_chunk_elems() { return b200::rs_chunk_elems(); }
int64_t rs_chunk_vecs() { return b200::rs_chunk_vecs(); }

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "vit_10b_fsdp_example_b200 native sm_90a kernels";
    m.def("gemm", &gemm);
    m.def("layernorm_fwd", &layernorm_fwd);
    m.def("layernorm_bwd", &layernorm_bwd);
    m.def("softmax_fwd", &softmax_fwd);
    m.def("softmax_bwd", &softmax_bwd);
    namespace py = pybind11;
    m.def("attention_fwd", &attention_fwd, py::arg("qkv"), py::arg("out"), py::arg("lse"), py::arg("probs"), py::arg("B"),
          py::arg("N"), py::arg("H"), py::arg("hd"), py::arg("drop_p") = 0.0, py::arg("drop_key") = 0);
    m.def("attention_supported", &attention_supported);
    m.def("attention_bwd", &attention_bwd, py::arg("qkv"), py::arg("dout"), py::arg("out"), py::arg("lse"),
          py::arg("delta"), py::arg("dqkv"), py::arg("colsum"), py::arg("B"), py::arg("N"), py::arg("H"), py::arg("hd"),
          py::arg("drop_p") = 0.0, py::arg("drop_key") = 0);
    m.def("cross_entropy", &cross_entropy, py::arg("logits"), py::arg("target"), py::arg("dlogits"), py::arg("loss"),
          py::arg("correct"), py::arg("lam") = 1.0, py::arg("smoothing") = 0.0);
    m.def("im2col", &im2col, py::arg("img"), py::arg("cols"), py::arg("P"), py::arg("lam") = py::none(),
          py::arg("box") = std::vector<int64_t>());
    m.def("gelu_fwd", &gelu_fwd);
    m.def("dgelu_mul", &dgelu_mul);
    m.def("swiglu_fwd", &swiglu_fwd);
    m.def("swiglu_bwd", &swiglu_bwd);
    m.def("dropout", &dropout);
    m.def("drop_path_scale", &drop_path_scale);
    m.def("drop_path_bwd", &drop_path_bwd);
    m.def("meanpool_fwd", &meanpool_fwd);
    m.def("meanpool_bwd", &meanpool_bwd);
    m.def("qk_norm_fwd", &qk_norm_fwd);
    m.def("qk_norm_bwd", &qk_norm_bwd);
    m.def("layer_scale_fold", &layer_scale_fold);
    m.def("layer_scale_bwd", &layer_scale_bwd);
    m.def("tokens_fwd", &tokens_fwd);
    m.def("tokens_bwd", &tokens_bwd);
    m.def("patch_drop_select", &patch_drop_select);
    m.def("im2col_gather", &im2col_gather, py::arg("img"), py::arg("keep"), py::arg("cols"), py::arg("P"),
          py::arg("lam") = py::none(), py::arg("box") = std::vector<int64_t>{});
    m.def("pos_gather", &pos_gather);
    m.def("patch_drop_bwd", &patch_drop_bwd);
    m.def("colsum", &colsum);
    m.def("sumsq", &sumsq);
    m.def("adamw_split", &adamw_split, py::arg("hi"), py::arg("lo"), py::arg("m"), py::arg("v"), py::arg("grad"),
          py::arg("clip_coef"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("wd"),
          py::arg("step"), py::arg("hyper") = py::none(), py::arg("ema_hi") = py::none(),
          py::arg("ema_lo") = py::none(), py::arg("ema_decay") = 0.0, py::arg("groups") = py::none(),
          py::arg("group_hyper") = py::none());
    m.def("adamw_fp32", &adamw_fp32, py::arg("w"), py::arg("m"), py::arg("v"), py::arg("grad"), py::arg("clip_coef"),
          py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("wd"), py::arg("step"),
          py::arg("ema") = py::none(), py::arg("ema_decay") = 0.0, py::arg("groups") = py::none(),
          py::arg("group_hyper") = py::none());
    m.def("split_fp32", &split_fp32);
    m.def("merge_fp32", &merge_fp32);
    m.def("clip_coef", &clip_coef);
    m.def("p2p_all_gather", &p2p_all_gather);
    m.def("ce_all_gather", &ce_all_gather);
    m.def("reduce_scatter", &reduce_scatter, py::arg("peer_ptrs"), py::arg("mc_ptr"), py::arg("rank"), py::arg("world"),
          py::arg("out"), py::arg("seg_table"), py::arg("total_chunks"), py::arg("in_is_bf16"), py::arg("scale"),
          py::arg("sumsq_out"), py::arg("max_ctas"), py::arg("sync"), py::arg("flag_ptrs"), py::arg("seq_dev"),
          py::arg("cta_ctr"), py::arg("hi"), py::arg("lo"), py::arg("m"), py::arg("v"), py::arg("hyper"),
          py::arg("groups") = py::none(), py::arg("group_hyper") = py::none());
    m.def("all_reduce_mean", &all_reduce_mean);
    m.def("rs_chunk_vecs", &rs_chunk_vecs);
    m.def("signal_barrier", &signal_barrier);
    m.def("allreduce_scalars", &allreduce_scalars);
    m.def("ag_chunk_bytes", &ag_chunk_bytes);
    m.def("rs_chunk_elems", &rs_chunk_elems);
}
