"""sm_90a implementation of the functional op set (same contract as ``torch_ops``).

Every function launches hand-written kernels from ``_C.so``:
  * GEMMs: persistent warp-specialised wgmma kernel (TMA ring, register accumulators) with fused epilogues
    (bias / GELU / dGELU / residual / pre-activation side output / bias-gradient column sums);
    forward (NT), dgrad (NN) and wgrad (TN) run on the same kernel via K-major / MN-major descriptors.
  * attention core: fused wgmma forward (keeps the row log-sum-exp) + fused backward kernels that read q/k/v in
    place from the packed qkv buffer through 4-D TMA tensor maps; scores never reach HBM, attention dropout included
    (the kernels regenerate the Philox mask of ``dropout`` in registers).  The un-fused path (batched wgmma GEMMs +
    softmax / softmax-backward kernels with materialised P) remains for B200_FUSED_ATTN_BWD=0 and unsupported shapes.
  * LayerNorm fwd/bwd, cross-entropy, im2col, column sums, sum of squares, fused AdamW.
  * QK normalisation: per-head LayerNorm of q and k on the packed qkv buffer and its backward (``qk_norm_fwd`` /
    ``qk_norm_bwd``, csrc/qk_norm.cu).
  * LayerScale: the per-channel branch scale folded into the proj / fc2 weight and bias, and its backward on the
    weight gradient (``layer_scale_fold`` / ``layer_scale_bwd``, csrc/layer_scale.cu).
  * prefix tokens: the class / register tokens put in front of every image's patch rows, and the backward that splits
    the token gradient into the patch rows and the per-token batch sums (``tokens_fwd`` / ``tokens_bwd``,
    csrc/prefix_tokens.cu).
  * SwiGLU: the gate silu(u[:, :Hd/2]) * u[:, Hd/2:] in the fc1 GEMM epilogue and its gradient in the fc2 dgrad
    epilogue (ACT_SWIGLU / ACT_DSWIGLU), and the memory-bound ``swiglu_fwd`` / ``swiglu_bwd`` for short K, the
    re-materialisation of g in backward and the MLP-dropout route.
  * patch dropout: the per-image kept-patch selection, the im2col of the kept patches, their position rows and the
    backward of the kept-token assembly (``patch_drop_select`` / ``patch_im2col(keep=)`` / ``pos_gather`` /
    ``patch_drop_bwd``, csrc/patch_drop.cu).
  * stochastic depth: per-sample Philox scales (``drop_path_scale``), applied as a row scale in the proj / fc2 GEMM
    epilogues, and ``drop_path_bwd`` (scaled branch gradient + its bias gradient in one pass).

What each group replaces in the reference (all of it reached through timm / torch_xla there):
  linear_fwd / dgrad / wgrad      nn.Linear in timm Attention.qkv / proj, Mlp.fc1 / fc2, the head (run_vit_training.py:134-141,153)
  attention_fwd / attention_bwd   timm Attention's softmax(q k^T * hd^-0.5) v with materialised scores (:134)
  ln_fwd / ln_bwd                 nn.LayerNorm in timm Block (eps 1e-5) and the final norm (:151, eps 1e-6)
  patch_im2col + linear_fwd       timm PatchEmbed conv k = s = P plus the pos_embed add (:124-129,156)
  cross_entropy                   nn.CrossEntropyLoss (:229,262) and the eval argmax/eq (:312-313)
  adamw_* / sumsq / clip_coef     torch.optim.AdamW (:237,278) and FSDP.clip_grad_norm_ (:270)

bf16 activations / weights, fp32 accumulation and statistics.  There is no PyTorch fallback here: if the
extension is missing this module fails to import on purpose.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import native

NAME = "sm100"


class _CountingModule:
    """Proxy over the native module that counts kernel launches (every entry point launches exactly one
    hand-written kernel); ``launch_count()`` feeds the ``gpu_launches`` field of bench.py."""

    def __init__(self, mod):
        object.__setattr__(self, "_mod", mod)
        object.__setattr__(self, "count", 0)

    def __getattr__(self, name):
        fn = getattr(self._mod, name)
        if not callable(fn):
            return fn

        def wrapped(*a, **k):
            object.__setattr__(self, "count", self.count + 1)
            return fn(*a, **k)

        object.__setattr__(self, name, wrapped)
        return wrapped


_C = _CountingModule(native.load())


def launch_count() -> int:
    return _C.count

ACT_NONE, ACT_GELU, ACT_DGELU, ACT_SWIGLU, ACT_DSWIGLU = 0, 1, 2, 3, 4
# GELU / dGELU are fused into the GEMM epilogue only when the reduction is deep enough to hide the math
# (ViT-10B: K = 5120 fused; ViT-L: K = 1024 -> plain GEMM + stand-alone elementwise kernel; the threshold has not
# been re-measured on H100)
import os as _os

FUSE_ACT_MIN_K = int(_os.environ.get("B200_FUSE_ACT_MIN_K", "2048"))
# SwiGLU routes, chosen by tools/bench_swiglu.py (H100 80GB HBM3, 700 W, 32768 rows; numbers in DESIGN.md):
#   fc1 forward: the fused epilogue took 0.69x (K = D = 1536) and 0.89x (K = 5120) the time of GEMM + swiglu_fwd
#   fc2 dgrad:   the fused epilogue took 0.85x at K = D = 1536 but 1.14x at K = 5120 the time of GEMM + swiglu_bwd +
#                colsum, so it runs only for K in the measured-faster range
SWIGLU_FWD_MIN_K = 1536
SWIGLU_DGRAD_K = (1536, 2048)

# SM carve-out for compute kernels while a communication kernel runs next to them (0 = all SMs).
_max_ctas = 0


def set_compute_max_ctas(n: int) -> None:
    global _max_ctas
    _max_ctas = int(n)


# GEMM CTA-cluster size: 0 = auto (one CTA per tile, see gemm_bf16), 1 or 2 (CTA pairs sharing the B tile) forced.
_gemm_cluster = 0


def set_gemm_cluster(n: int) -> None:
    global _gemm_cluster
    assert n in (0, 1, 2), n
    _gemm_cluster = int(n)


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "expected a row-major 2-D (possibly strided) matrix"
    return t.stride(0)


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def _tma_rows(t: torch.Tensor) -> torch.Tensor:
    """TMA needs 16-byte row strides and base.  Matrices whose width is not a multiple of 8 (e.g. a classifier
    with an odd class count) are copied into a zero-padded buffer and used through a strided view."""
    if t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0:
        return t
    rows, cols = t.shape
    buf = torch.zeros(rows, _pad8(cols), dtype=t.dtype, device=t.device)
    buf[:, :cols].copy_(t)
    return buf[:, :cols]


def _bias_ok(b: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """The epilogue reads bias in 16-byte vectors: pad odd-length biases so the tail read stays in bounds."""
    if b is None or b.numel() % 8 == 0:
        return b
    buf = torch.zeros(_pad8(b.numel()), dtype=b.dtype, device=b.device)
    buf[: b.numel()].copy_(b)
    return buf


def gemm_raw(a, lda, major_a, b, ldb, major_b, d, ldd, M, N, K, *, bias=None, residual=None, ld_res=0,
             res_row_mod=0, aux_in=None, ld_aux=0, aux_out=None, ld_aux_out=0, colsum=None, colsum_bi_stride=0,
             act=ACT_NONE, batch=(), block_n=0, cluster=None, max_ctas=None, ag=(), row_scale=None, rows_per_scale=0):
    _C.gemm(a, lda, major_a, b, ldb, major_b, d, ldd, M, N, K, bias, residual, ld_res, res_row_mod, aux_in, ld_aux,
            aux_out, ld_aux_out, colsum, colsum_bi_stride, act, list(batch), block_n,
            _gemm_cluster if cluster is None else cluster, _max_ctas if max_ctas is None else max_ctas, list(ag),
            row_scale, rows_per_scale)


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def ln_fwd(x, w, b, eps: float):
    rows = x.shape[0]
    y = torch.empty_like(x)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    _C.layernorm_fwd(x, w, b, y, mean, rstd, eps)
    return y, mean, rstd


def ln_bwd(dy, x, w, mean, rstd, dres=None, want_dxsum: bool = False):
    D = x.shape[1]
    dx = torch.empty_like(x)
    acc = torch.zeros(3 if want_dxsum else 2, D, dtype=torch.float32, device=x.device)
    _C.layernorm_bwd(dy, x, w, mean, rstd, dres, dx, acc[0], acc[1], acc[2] if want_dxsum else None)
    return dx, acc[0], acc[1], (acc[2] if want_dxsum else None)


# ------------------------------------------------------------------------------------------------
# QK normalisation (csrc/qk_norm.cu): per-head LayerNorm of q and k on the packed qkv buffer
# ------------------------------------------------------------------------------------------------
def qk_norm_fwd(qkv, H: int, hd: int, wq, bq, wk, bk, eps: float, inplace: bool = False):
    """Returns (out, mean, rstd): out = qkv with every q head normalised over hd (weight wq, bias bq) and every k head
    (wk, bk), v unchanged; mean / rstd fp32 [T * 2 * H].  inplace=True writes into qkv itself (the v columns are not
    touched) and returns it; otherwise out is a new [T, 3D] buffer that also receives a copy of v."""
    T = qkv.shape[0]
    out = qkv if inplace else torch.empty(T, 3 * H * hd, dtype=qkv.dtype, device=qkv.device)
    mean = torch.empty(T * 2 * H, dtype=torch.float32, device=qkv.device)
    rstd = torch.empty(T * 2 * H, dtype=torch.float32, device=qkv.device)
    _C.qk_norm_fwd(qkv, wq, bq, wk, bk, out, mean, rstd, H, hd, float(eps))
    return out, mean, rstd


def qk_norm_bwd(dqkv, qkv, H: int, hd: int, wq, wk, mean, rstd):
    """In place on dqkv[:, 0:2D); returns (dqkv, dwq, dbq, dwk, dbk, colsum[2D]) like ``torch_ops.qk_norm_bwd``."""
    acc = torch.zeros(4 * hd + 2 * H * hd, dtype=torch.float32, device=qkv.device)
    dwq, dbq, dwk, dbk = acc[:4 * hd].view(4, hd)
    cs = acc[4 * hd:]
    _C.qk_norm_bwd(dqkv, qkv, wq, wk, mean, rstd, dwq, dbq, dwk, dbk, cs, H, hd)
    return dqkv, dwq, dbq, dwk, dbk, cs


# ------------------------------------------------------------------------------------------------
# LayerScale (csrc/layer_scale.cu): per-channel branch scale folded into the proj / fc2 weight and bias
# ------------------------------------------------------------------------------------------------
def layer_scale_fold(W, b, gamma):
    """(Wg, bg) = (bf16(gamma_c * W[c, :]), bf16(gamma_c * b_c)) like ``torch_ops.layer_scale_fold``."""
    Wg = torch.empty_like(W, memory_format=torch.contiguous_format)
    bg = torch.empty_like(b, memory_format=torch.contiguous_format)
    _C.layer_scale_fold(W, b, gamma, Wg, bg)
    return Wg, bg


def layer_scale_bwd(W, b, gamma, dW, S):
    """In place on dW (M in, gamma o M out); returns (Wg, db, dgamma) like ``torch_ops.layer_scale_bwd``."""
    Wg = torch.empty_like(W, memory_format=torch.contiguous_format)
    out = torch.empty(2, W.shape[0], dtype=torch.float32, device=W.device)
    _C.layer_scale_bwd(W, b, gamma, dW, S, Wg, out[0], out[1])
    return Wg, out[0], out[1]


# ------------------------------------------------------------------------------------------------
# Prefix tokens (csrc/prefix_tokens.cu): class and register tokens in front of every image's patch rows
# ------------------------------------------------------------------------------------------------
def tokens_fwd(y, cls, reg, pos, B: int, N: int):
    """x0 [B * (N + P), D] like ``torch_ops.tokens_fwd`` (reg None when there are no register tokens)."""
    D = y.shape[1]
    P = 1 + (reg.numel() // D if reg is not None else 0)
    x0 = torch.empty(B * (N + P), D, dtype=y.dtype, device=y.device)
    _C.tokens_fwd(y, cls, reg, pos, x0, B, N)
    return x0


def tokens_bwd(dx0, B: int, N: int, P: int):
    """(dpatch [B * N, D] bf16, dtok [N + P, D] fp32) in one pass, like ``torch_ops.tokens_bwd``; dtok is summed over
    the batch in a fixed order (the same bits in every run)."""
    D = dx0.shape[1]
    dpatch = torch.empty(B * N, D, dtype=dx0.dtype, device=dx0.device)
    dtok = torch.empty(N + P, D, dtype=torch.float32, device=dx0.device)
    _C.tokens_bwd(dx0, dpatch, dtok, B, N, P)
    return dpatch, dtok


# ------------------------------------------------------------------------------------------------
# Patch dropout (csrc/patch_drop.cu): every image keeps K of its N patches in a training step
# ------------------------------------------------------------------------------------------------
def patch_drop_select(key: int, B: int, N: int, K: int, offset: int, device):
    """(keep int32 [B, K], inv int32 [B, N]) with the bits of ``torch_ops.patch_drop_select``."""
    keep = torch.empty(B, K, dtype=torch.int32, device=device)
    inv = torch.empty(B, N, dtype=torch.int32, device=device)
    _C.patch_drop_select(keep, inv, int(N), int(K), int(offset), _drop_key(key))
    return keep, inv


def pos_gather(pos, keep):
    """[B * K, D]: the position rows pos[keep[b, i]] of the kept patches."""
    out = torch.empty(keep.numel(), pos.shape[1], dtype=pos.dtype, device=pos.device)
    _C.pos_gather(pos.contiguous(), keep, out)
    return out


def patch_drop_bwd(dx0, inv, B: int, N: int, K: int, P: int):
    """(dpatch [B * K, D] bf16 or None when P == 0, dtok [P + N, D] fp32) in one pass, like
    ``torch_ops.patch_drop_bwd``; dtok is summed over the batch in a fixed order (the same bits in every run)."""
    D = dx0.shape[1]
    dpatch = torch.empty(B * K, D, dtype=dx0.dtype, device=dx0.device) if P else None
    dtok = torch.empty(P + N, D, dtype=torch.float32, device=dx0.device)
    _C.patch_drop_bwd(dx0, inv, dpatch, dtok, B, N, K, P)
    return dpatch, dtok


# ------------------------------------------------------------------------------------------------
# Linear
# ------------------------------------------------------------------------------------------------
def linear_fwd(x, w, bias=None, act: Optional[str] = None, residual=None, res_row_mod: int = 0,
               want_preact: bool = False, ag=None, row_scale=None, rows_per_scale: int = 0):
    """ag: optional all-gather fusion spec (see Sm100Backend.ag_fuse_spec): the kernel itself pulls the peers'
    shards of `w` over NVLink while it computes.
    row_scale: fp32 [M / rows_per_scale] per-sample scales (stochastic depth), applied in the epilogue as
    (x w^T + bias) * row_scale[m / rows_per_scale] before the residual add; only without an activation."""
    M, K = x.shape
    N = w.shape[0]
    if act == "swiglu":
        return _linear_swiglu(x, w, bias, residual, want_preact, ag, row_scale)
    if row_scale is not None:
        assert act is None and not want_preact and rows_per_scale > 0, "row_scale: plain linear layers only"
        assert row_scale.dtype == torch.float32 and row_scale.numel() * rows_per_scale == M, "one scale per sample"
    if act == "gelu" and K < FUSE_ACT_MIN_K and N % 8 == 0 and ag is None:
        # short K: the activation math would not fit under a tile's MMA time -> plain GEMM + memory-bound GELU
        pre = linear_fwd(x, w, bias, residual=None)
        y = torch.empty_like(pre)
        _C.gelu_fwd(pre, y)
        if residual is not None:
            y += residual
        return (y, pre) if want_preact else y
    x, w = _tma_rows(x), _tma_rows(w)
    ldy = _pad8(N)
    y = torch.empty(M, ldy, dtype=x.dtype, device=x.device)
    pre = torch.empty(M, ldy, dtype=x.dtype, device=x.device) if want_preact else None
    gemm_raw(x, _ld(x), 0, w, _ld(w), 0, y, ldy, M, N, K, bias=_bias_ok(bias), residual=residual,
             ld_res=_ld(residual) if residual is not None else 0, res_row_mod=res_row_mod, aux_out=pre,
             ld_aux_out=ldy, act=ACT_GELU if act == "gelu" else ACT_NONE, ag=ag or (), row_scale=row_scale,
             rows_per_scale=rows_per_scale)
    if ldy != N:
        y = y[:, :N].contiguous()
        pre = pre[:, :N].contiguous() if pre is not None else None
    return (y, pre) if want_preact else y


def _linear_swiglu(x, w, bias, residual, want_preact: bool, ag, row_scale):
    """act="swiglu" (w: the packed [Hd, K] fc1 weight): g [M, Hd / 2], and the pre-activation u [M, Hd] if wanted.
    The GEMM tiles pair fc1 rows n and Hd / 2 + n, so the gate runs in registers; at short K the plain GEMM and
    ``swiglu_fwd`` run instead (SWIGLU_FWD_MIN_K)."""
    assert residual is None and row_scale is None, "swiglu: no residual or row scale"
    M, K = x.shape
    Hd = w.shape[0]
    if Hd % 16 != 0:
        raise ValueError(f"swiglu: the fc1 width Hd must be a multiple of 16, got {Hd}")
    if K < SWIGLU_FWD_MIN_K and ag is None:
        pre = linear_fwd(x, w, bias)
        g = swiglu_fwd(pre)
        return (g, pre) if want_preact else g
    x, w = _tma_rows(x), _tma_rows(w)
    g = torch.empty(M, Hd // 2, dtype=x.dtype, device=x.device)
    pre = torch.empty(M, Hd, dtype=x.dtype, device=x.device) if want_preact else None
    gemm_raw(x, _ld(x), 0, w, _ld(w), 0, g, Hd // 2, M, Hd // 2, K, bias=bias, aux_out=pre, ld_aux_out=Hd,
             act=ACT_SWIGLU, ag=ag or ())
    return (g, pre) if want_preact else g


def linear_dgrad(dy, w, dgelu_preact=None, want_colsum: bool = False, dswiglu_preact=None):
    """dswiglu_preact = u [M, Hd]: returns du = [dh * value * silu'(gate) | dh * silu(gate)] [M, Hd] for
    dh = dy @ w [M, Hd / 2] (like ``torch_ops.linear_dgrad``): from the fc2 dgrad epilogue where that measured faster
    (SWIGLU_DGRAD_K over the reduction depth N = D), else the plain dgrad + ``swiglu_bwd`` + ``colsum``."""
    M, N = dy.shape
    K = w.shape[1]
    if dswiglu_preact is not None:
        u = dswiglu_preact
        if not SWIGLU_DGRAD_K[0] <= N <= SWIGLU_DGRAD_K[1]:
            du = swiglu_bwd(linear_dgrad(dy, w), u)
            return (du, colsum(du)) if want_colsum else du
        dy, w = _tma_rows(dy), _tma_rows(w)
        du = torch.empty(M, 2 * K, dtype=dy.dtype, device=dy.device)
        cs = torch.zeros(2 * K, dtype=torch.float32, device=dy.device) if want_colsum else None
        gemm_raw(dy, _ld(dy), 0, w, _ld(w), 1, du, 2 * K, M, K, N, aux_in=u, ld_aux=_ld(u), aux_out=du[:, K:],
                 ld_aux_out=2 * K, act=ACT_DSWIGLU, colsum=cs)
        return (du, cs) if want_colsum else du
    if dgelu_preact is not None and N < FUSE_ACT_MIN_K and K % 8 == 0:
        dx = linear_dgrad(dy, w)
        _C.dgelu_mul(dx, dgelu_preact, dx)
        if want_colsum:
            return dx, colsum(dx)
        return dx
    dy, w = _tma_rows(dy), _tma_rows(w)
    dx = torch.empty(M, K, dtype=dy.dtype, device=dy.device)
    cs = torch.zeros(K, dtype=torch.float32, device=dy.device) if want_colsum else None
    gemm_raw(dy, _ld(dy), 0, w, _ld(w), 1, dx, K, M, K, N, aux_in=dgelu_preact,
             ld_aux=_ld(dgelu_preact) if dgelu_preact is not None else 0,
             act=ACT_DGELU if dgelu_preact is not None else ACT_NONE, colsum=cs)
    return (dx, cs) if want_colsum else dx


def linear_wgrad(dy, x, out=None, block_n: int = 0):
    T, N = dy.shape
    K = x.shape[1]
    dy, x = _tma_rows(dy), _tma_rows(x)
    if out is None:
        out = torch.empty(N, K, dtype=dy.dtype, device=dy.device)
    gemm_raw(dy, _ld(dy), 1, x, _ld(x), 1, out, _ld(out), N, K, T, block_n=block_n)
    return out


def gelu_fwd(u):
    g = torch.empty_like(u)
    _C.gelu_fwd(u, g)
    return g


def dgelu_mul(dg, u):
    du = torch.empty_like(dg)
    _C.dgelu_mul(dg.contiguous(), u, du)
    return du


def swiglu_fwd(u):
    """g [M, Hd / 2] = silu(u[:, :Hd/2]) * u[:, Hd/2:] (csrc/elementwise.cu), like ``torch_ops.swiglu_fwd``."""
    u = u.contiguous()
    g = torch.empty(u.shape[0], u.shape[1] // 2, dtype=u.dtype, device=u.device)
    _C.swiglu_fwd(u, g)
    return g


def swiglu_bwd(dg, u):
    """du [M, Hd] = [dg * value * silu'(gate) | dg * silu(gate)], like ``torch_ops.swiglu_bwd``."""
    u = u.contiguous()
    du = torch.empty_like(u)
    _C.swiglu_bwd(dg.contiguous(), u, du)
    return du


def colsum(x):
    out = torch.zeros(x.shape[1], dtype=torch.float32, device=x.device)
    _C.colsum(x, out)
    return out


# ------------------------------------------------------------------------------------------------
# Attention core
# ------------------------------------------------------------------------------------------------
FUSED_ATTENTION = _os.environ.get("B200_FUSED_ATTN", "1") != "0"


def dropout(x, p: float, key: int):
    """Philox-keyed dropout kernel (csrc/elementwise.cu): the mask is a function of (key, position), never stored."""
    xc = x.contiguous()
    assert xc.numel() % 8 == 0, "dropout kernel works on whole 16-byte vectors"
    y = torch.empty_like(xc)
    _C.dropout(xc, y, float(p), _drop_key(key))
    return y


def drop_path_scale(key: int, p: float, B: int, offset: int, device):
    """Stochastic depth: fp32 [B], entry b = 0 (sample offset + b dropped) or dropout_scale (kept).  Same bits as
    ``torch_ops.drop_path_scale``."""
    scale = torch.empty(B, dtype=torch.float32, device=device)
    _C.drop_path_scale(scale, int(offset), float(p), _drop_key(key))
    return scale


def drop_path_bwd(dy, scale, N: int):
    """(dt = bf16(scale[row / N] * dy), fp32 column sums of dt) in one pass."""
    dyc = dy.contiguous()
    dt = torch.empty_like(dyc)
    cs = torch.zeros(dyc.shape[1], dtype=torch.float32, device=dyc.device)
    _C.drop_path_bwd(dyc, scale, dt, cs, int(N))
    return dt, cs


def mean_pool(xn, B: int, N: int):
    pooled = torch.empty(B, xn.shape[1], dtype=xn.dtype, device=xn.device)
    _C.meanpool_fwd(xn, pooled, B, N)
    return pooled


def mean_pool_bwd(dpooled, B: int, N: int):
    dxn = torch.empty(B * N, dpooled.shape[1], dtype=dpooled.dtype, device=dpooled.device)
    _C.meanpool_bwd(dpooled.contiguous(), dxn, B, N)
    return dxn


def _drop_key(key: int) -> int:
    return int(key) & 0x7FFFFFFFFFFFFFFF


def attention_fwd(qkv, B: int, N: int, H: int, hd: int, drop=None, need_p: bool = True):
    """Returns (out [B*N, D], P).  P = softmax probabilities [B*H, N, ldp] for the backward, or None when
    need_p=False and the fused kernel ran (scores never reach HBM then).
    drop = (p, key): attention dropout.  With need_p the probabilities are materialised (un-fused path), the dropped
    copy that feeds P V comes from the Philox dropout kernel and the returned P is the un-dropped one (backward
    regenerates the mask); without need_p the fused kernel applies the same mask in registers."""
    D = H * hd
    ldp = _pad8(N)
    if drop is not None and not need_p and FUSED_ATTENTION and _C.attention_supported(N, hd):
        out = torch.empty(B * N, D, dtype=qkv.dtype, device=qkv.device)
        _C.attention_fwd(qkv, out, None, None, B, N, H, hd, float(drop[0]), _drop_key(drop[1]))
        return out, None
    if drop is not None:
        p = attention_probs(qkv, B, N, H, hd)
        pd = dropout(p, drop[0], drop[1])
        out = torch.empty(B * N, D, dtype=qkv.dtype, device=qkv.device)
        ld3 = qkv.stride(0)
        gemm_raw(pd, ldp, 0, qkv[:, 2 * D:], ld3, 1, out, D, N, hd, N,
                 batch=(H, B, N * ldp, H * N * ldp, hd, N * ld3, hd, N * D))
        return out, p
    # Fused kernel (S and P live in registers).  With P requested it is still faster than GEMM + softmax + GEMM:
    # 1445 vs 1996 us at B128 N256 H32 hd160, 383 vs 654 us at B128 N196 H16 hd64 (CUDA events, H100 80GB HBM3, 700 W).
    if FUSED_ATTENTION and _C.attention_supported(N, hd):
        out = torch.empty(B * N, D, dtype=qkv.dtype, device=qkv.device)
        p = None
        if need_p:
            p = torch.empty(B * H, N, ldp, dtype=qkv.dtype, device=qkv.device)
            if ldp != N:
                p[:, :, N:].zero_()
        _C.attention_fwd(qkv, out, None, p, B, N, H, hd)
        return out, p
    p = torch.empty(B * H, N, ldp, dtype=qkv.dtype, device=qkv.device)
    if ldp != N:
        p[:, :, N:].zero_()
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    ld3 = qkv.stride(0)
    # S = Q K^T  (per (image, head) problem; operands addressed in place inside qkv)
    gemm_raw(q, ld3, 0, k, ld3, 0, p, ldp, N, N, hd,
             batch=(H, B, hd, N * ld3, hd, N * ld3, N * ldp, H * N * ldp))
    _C.softmax_fwd(p, B * H * N, N, ldp, hd ** -0.5)
    out = torch.empty(B * N, D, dtype=qkv.dtype, device=qkv.device)
    # O = P V  (V is MN-major: head-dim contiguous, keys strided)
    gemm_raw(p, ldp, 0, v, ld3, 1, out, D, N, hd, N,
             batch=(H, B, N * ldp, H * N * ldp, hd, N * ld3, hd, N * D))
    return out, p


# Fused (flash-style) forward + backward pair: the forward keeps only the row log-sum-exp, the backward kernels
# (csrc/attention_sm90.cu) rebuild P tile by tile; scores never reach HBM and no [B*H, N, N] buffer is allocated (at
# the ViT-10B shape P alone would be 512 MiB per block).  Fused by default; B200_FUSED_ATTN_BWD=0 selects the un-fused path.
FLASH_ATTENTION = _os.environ.get("B200_FUSED_ATTN_BWD", "") != "0"


def flash_supported(N: int, hd: int) -> bool:
    return bool(_C.attention_supported(N, hd))


def use_flash(N: int, hd: int) -> bool:
    """Model-level policy: run the attention core through the fused forward (log-sum-exp) + fused backward pair?"""
    return FLASH_ATTENTION and flash_supported(N, hd)


def attention_fwd_lse(qkv, B: int, N: int, H: int, hd: int, drop=None):
    """drop = (p, key): attention dropout with exactly the mask ``dropout(P, p, key)`` would draw for the [B*H, N, ldp]
    probability buffer of the un-fused path; lse stays that of the undropped scores."""
    out = torch.empty(B * N, H * hd, dtype=qkv.dtype, device=qkv.device)
    lse = torch.empty(B * H, N, dtype=torch.float32, device=qkv.device)
    p, key = drop if drop is not None else (0.0, 0)
    _C.attention_fwd(qkv, out, lse, None, B, N, H, hd, float(p), _drop_key(key))
    return out, lse


def attention_bwd_lse(dout, qkv, out, lse, B: int, N: int, H: int, hd: int, want_colsum: bool = False, drop=None):
    """drop: the (p, key) of the forward; the kernels regenerate its mask."""
    dqkv = torch.empty(B * N, 3 * H * hd, dtype=qkv.dtype, device=qkv.device)
    delta = torch.empty(B * H, N, dtype=torch.float32, device=qkv.device)  # scratch: rowsum(dO o O)
    # the backward kernels reduce the qkv bias gradient (column sums of dq | dk | dv) from their epilogue tiles
    cs = torch.zeros(3 * H * hd, dtype=torch.float32, device=qkv.device) if want_colsum else None
    p, key = drop if drop is not None else (0.0, 0)
    _C.attention_bwd(qkv, dout, out, lse, delta, dqkv, cs, B, N, H, hd, float(p), _drop_key(key))
    return (dqkv, cs) if want_colsum else dqkv


def attention_probs(qkv, B: int, N: int, H: int, hd: int):
    """P = softmax(Q K^T / sqrt(hd)) alone: re-materialised in backward for blocks that kept only qkv."""
    D = H * hd
    ldp = _pad8(N)
    p = torch.empty(B * H, N, ldp, dtype=qkv.dtype, device=qkv.device)
    if ldp != N:
        p[:, :, N:].zero_()
    ld3 = qkv.stride(0)
    gemm_raw(qkv[:, :D], ld3, 0, qkv[:, D:2 * D], ld3, 0, p, ldp, N, N, hd,
             batch=(H, B, hd, N * ld3, hd, N * ld3, N * ldp, H * N * ldp))
    _C.softmax_fwd(p, B * H * N, N, ldp, hd ** -0.5)
    return p


def attention_bwd(dout, qkv, p, B: int, N: int, H: int, hd: int, want_colsum: bool = False, drop=None):
    """drop = (p, key) of the forward: the dropped probabilities (for dV) and the mask on dP are regenerated."""
    D = H * hd
    ldp = p.shape[2]
    ld3 = qkv.stride(0)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    dqkv = torch.empty(B * N, 3 * D, dtype=qkv.dtype, device=qkv.device)
    dq, dk, dv = dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]
    cs = torch.zeros(3 * D, dtype=torch.float32, device=qkv.device) if want_colsum else None
    ldo = dout.stride(0)
    bp = (N * ldp, H * N * ldp)      # batch strides of P-shaped buffers
    bq = (hd, N * ld3)               # ... of q/k/v inside qkv
    bo = (hd, N * ldo)
    bd = (hd, N * 3 * D)             # ... of dq/dk/dv inside dqkv
    # dV = P^T dO   (with attention dropout: the dropped P that fed the forward P V)
    pv = p if drop is None else dropout(p, drop[0], drop[1])
    gemm_raw(pv, ldp, 1, dout, ldo, 1, dv, 3 * D, N, hd, N, batch=(H, B, *bp, *bo, *bd),
             colsum=cs[2 * D:] if want_colsum else None, colsum_bi_stride=hd)
    del pv
    # dP = dO V^T
    dp = torch.empty_like(p)
    if ldp != N:
        dp[:, :, N:].zero_()
    gemm_raw(dout, ldo, 0, v, ld3, 0, dp, ldp, N, N, hd, batch=(H, B, *bo, *bq, *bp))
    if drop is not None:
        _C.dropout(dp, dp, float(drop[0]), _drop_key(drop[1]))  # same key and shape -> same mask
    # dS = scale * P * (dP - rowsum(dP * P))   (in place)
    _C.softmax_bwd(dp, p, B * H * N, N, ldp, hd ** -0.5)
    # dQ = dS K ; dK = dS^T Q
    gemm_raw(dp, ldp, 0, k, ld3, 1, dq, 3 * D, N, hd, N, batch=(H, B, *bp, *bq, *bd),
             colsum=cs[:D] if want_colsum else None, colsum_bi_stride=hd)
    gemm_raw(dp, ldp, 1, q, ld3, 1, dk, 3 * D, N, hd, N, batch=(H, B, *bp, *bq, *bd),
             colsum=cs[D:2 * D] if want_colsum else None, colsum_bi_stride=hd)
    return (dqkv, cs) if want_colsum else dqkv


# ------------------------------------------------------------------------------------------------
# Patch embedding, loss
# ------------------------------------------------------------------------------------------------
def patch_im2col(images, P: int, kpad: int, dtype, mix=None, keep=None):
    """mix = (lam, box) from vit.draw_mix: Mixup (box None) or CutMix of image b with image B-1-b, fused into the
    im2col (torch_ops.mix_images is the reference).  keep [B, K] (patch dropout): only the kept patches, by the
    gathering im2col kernel."""
    B, _, S, _ = images.shape
    if keep is not None:
        cols = torch.empty(keep.numel(), kpad, dtype=dtype, device=images.device)
        if mix is None:
            _C.im2col_gather(images.contiguous(), keep, cols, P)
        else:
            lam, box = mix
            _C.im2col_gather(images.contiguous(), keep, cols, P, float(lam), list(box) if box is not None else [])
        return cols
    G = S // P
    cols = torch.empty(B * G * G, kpad, dtype=dtype, device=images.device)
    if mix is None:
        _C.im2col(images.contiguous(), cols, P)
    else:
        lam, box = mix
        _C.im2col(images.contiguous(), cols, P, float(lam), list(box) if box is not None else [])
    return cols


def cross_entropy(logits, target, want_grad: bool = True, mix=None, smoothing: float = 0.0):
    """mix / smoothing: the soft target lam * smooth(y_b) + (1 - lam) * smooth(y_{B-1-b}) (timm mixup_target)."""
    loss = torch.zeros(1, dtype=torch.float32, device=logits.device)
    correct = torch.zeros(1, dtype=torch.int32, device=logits.device)
    dlogits = torch.empty_like(logits) if want_grad else None
    if mix is None and smoothing == 0:
        _C.cross_entropy(logits, target, dlogits, loss, correct)
    else:
        lam = 1.0 if mix is None else float(mix[0])
        _C.cross_entropy(logits, target, dlogits, loss, correct, lam, float(smoothing))
    return loss[0], dlogits, correct[0]


# ------------------------------------------------------------------------------------------------
# Optimizer pieces
# ------------------------------------------------------------------------------------------------
def sumsq(x, out):
    _C.sumsq(x, out)


def clip_coef(sumsq_t, max_norm: float):
    coef = torch.empty(1, dtype=torch.float32, device=sumsq_t.device)
    norm = torch.empty(1, dtype=torch.float32, device=sumsq_t.device)
    _C.clip_coef(sumsq_t, max_norm, coef, norm)
    return coef, norm


def adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step: int, ema=None, ema_decay: float = 0.0,
               groups=None, group_hyper=None):
    """ema: optional fp32 model EMA, updated in the same pass as ema = fmaf(d, ema, (1 - d) * w_new).
    groups / group_hyper: optional parameter groups, the uint8 group of every 64-element chunk and the fp32 [G, 2]
    rows of (lr_scale, wd); the grouped kernels then use lr * lr_scale and that wd per chunk (`wd` is unused)."""
    if groups is not None:
        _C.adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, ema, float(ema_decay), groups, group_hyper)
    elif ema is None:
        _C.adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step)
    else:
        _C.adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, ema, float(ema_decay))


def adamw_split(hi, lo, m, v, grad, clip, lr, beta1, beta2, eps, wd, step: int, hyper=None, ema=None,
                ema_decay: float = 0.0, groups=None, group_hyper=None):
    """hyper: optional device tensor [lr, step] that overrides the host scalars (CUDA-graph replay).
    ema: optional (ema_hi, ema_lo), the model EMA in the master's split form, updated in the same pass as
    ema = fmaf(d, ema, (1 - d) * w_new) with d = ema_decay.  groups / group_hyper: as in adamw_fp32."""
    if groups is not None:
        e_hi, e_lo = ema if ema is not None else (None, None)
        _C.adamw_split(hi, lo, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, hyper, e_hi, e_lo,
                       float(ema_decay), groups, group_hyper)
    elif ema is None:
        _C.adamw_split(hi, lo, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, hyper)
    else:
        _C.adamw_split(hi, lo, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, hyper, ema[0], ema[1],
                       float(ema_decay))


def split_fp32(w, hi, lo):
    _C.split_fp32(w, hi, lo)


def merge_fp32(hi, lo, w):
    _C.merge_fp32(hi, lo, w)
