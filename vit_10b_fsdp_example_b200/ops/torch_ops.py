"""Reference implementation of the functional op set in plain PyTorch.

This is (a) the CPU / gloo test backend, (b) the fp32 numerical oracle every sm_90a kernel is tested
against, and (c) the semantics contract for ``cuda_ops``.  Every function here has a same-named,
same-signature twin in ``cuda_ops`` that runs the hand-written kernels.

All matrices are 2-D ``[tokens, features]``; the model code does its own reshapes.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

NAME = "torch"


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t if t.dtype == torch.float32 else t.float()


# ------------------------------------------------------------------------------------------------
# LayerNorm (timm Block.norm1 / norm2, final norm) -- reference run_vit_training.py:134-141,151
# ------------------------------------------------------------------------------------------------
def ln_fwd(x, w, b, eps: float):
    xf = _f32(x)
    mean = xf.mean(dim=-1)
    var = xf.var(dim=-1, unbiased=False)
    rstd = torch.rsqrt(var + eps)
    y = (xf - mean[:, None]) * rstd[:, None] * _f32(w) + _f32(b)
    return y.to(x.dtype), mean, rstd


def ln_bwd(dy, x, w, mean, rstd, dres=None, want_dxsum: bool = False):
    """Returns dx (= dres + LN backward), dw fp32, db fp32, colsum(dx) fp32 or None."""
    dyf, xf, wf = _f32(dy), _f32(x), _f32(w)
    xhat = (xf - mean[:, None]) * rstd[:, None]
    g = dyf * wf
    s1 = g.mean(dim=-1, keepdim=True)
    s2 = (g * xhat).mean(dim=-1, keepdim=True)
    dx = rstd[:, None] * (g - s1 - xhat * s2)
    if dres is not None:
        dx = dx + _f32(dres)
    dw = (dyf * xhat).sum(dim=0)
    db = dyf.sum(dim=0)
    dx = dx.to(x.dtype)
    dxsum = _f32(dx).sum(dim=0) if want_dxsum else None
    return dx, dw, db, dxsum


# ------------------------------------------------------------------------------------------------
# QK normalisation (timm Attention(qk_norm=True): q_norm / k_norm = nn.LayerNorm(head_dim) applied per head)
# qkv is the packed [T, 3D] projection (D = H * hd); statistics are indexed [T, 2, H] (q heads, then k heads).
# ------------------------------------------------------------------------------------------------
def qk_norm_fwd(qkv, H: int, hd: int, wq, bq, wk, bk, eps: float, inplace: bool = False):
    """Returns (out, mean, rstd): out = qkv with every q head normalised over hd (weight wq, bias bq) and every k head
    (wk, bk), v unchanged; mean / rstd fp32 [T * 2 * H].  inplace=True writes into qkv itself and returns it."""
    T, D = qkv.shape[0], H * hd
    x = _f32(qkv[:, : 2 * D]).reshape(T, 2, H, hd)
    mean = x.mean(dim=-1)
    rstd = torch.rsqrt(x.var(dim=-1, unbiased=False) + eps)
    w = torch.stack([_f32(wq), _f32(wk)])[None, :, None, :]
    b = torch.stack([_f32(bq), _f32(bk)])[None, :, None, :]
    y = ((x - mean[..., None]) * rstd[..., None] * w + b).reshape(T, 2 * D).to(qkv.dtype)
    out = qkv if inplace else qkv.clone()
    out[:, : 2 * D] = y
    return out, mean.reshape(-1), rstd.reshape(-1)


def qk_norm_bwd(dqkv, qkv, H: int, hd: int, wq, wk, mean, rstd):
    """LayerNorm backward of the q / k heads, in place on dqkv[:, 0:2D) (gradient of the normalised q / k in, of the
    un-normalised q / k out; dv untouched).  Returns (dqkv, dwq, dbq, dwk, dbk, colsum): fp32 [hd] parameter
    gradients summed over all T * H heads of each side, and fp32 [2D] column sums of the new (rounded) dq / dk, which
    are the q / k part of the qkv bias gradient."""
    T, D = qkv.shape[0], H * hd
    x = _f32(qkv[:, : 2 * D]).reshape(T, 2, H, hd)
    dy = _f32(dqkv[:, : 2 * D]).reshape(T, 2, H, hd)
    m, r = mean.view(T, 2, H, 1), rstd.view(T, 2, H, 1)
    xhat = (x - m) * r
    g = dy * torch.stack([_f32(wq), _f32(wk)])[None, :, None, :]
    dx = r * (g - g.mean(dim=-1, keepdim=True) - xhat * (g * xhat).mean(dim=-1, keepdim=True))
    dw = (dy * xhat).sum(dim=(0, 2))
    db = dy.sum(dim=(0, 2))
    dqkv[:, : 2 * D] = dx.reshape(T, 2 * D).to(dqkv.dtype)
    cs = _f32(dqkv[:, : 2 * D]).sum(dim=0)
    return dqkv, dw[0], db[0], dw[1], db[1], cs


# ------------------------------------------------------------------------------------------------
# LayerScale (timm LayerScale: x * gamma on a branch u = a W^T + b), folded into the layer's weight and bias
# ------------------------------------------------------------------------------------------------
def layer_scale_fold(W, b, gamma):
    """(Wg, bg) = (gamma_c * W[c, :], gamma_c * b_c), each rounded once to W's dtype: a Wg^T + bg = gamma o u."""
    g = _f32(gamma)
    return (_f32(W) * g[:, None]).to(W.dtype), (_f32(b) * g).to(b.dtype)


def layer_scale_bwd(W, b, gamma, dW, S):
    """dW holds M = dy'^T a (the wgrad of the un-scaled layer) and is overwritten with gamma o M; S = fp32 colsum(dy').
    Returns (Wg, db, dgamma): Wg as ``layer_scale_fold``, db = gamma o S and dgamma_c = sum_k W[c, k] M[c, k] + b_c S_c
    (= sum_r dy'[r, c] u[r, c]), both fp32 [D]."""
    g, m, s = _f32(gamma), _f32(dW), _f32(S)
    dgamma = (_f32(W) * m).sum(dim=1) + _f32(b) * s
    dW.copy_(m * g[:, None])
    return (_f32(W) * g[:, None]).to(W.dtype), g * s, dgamma


# ------------------------------------------------------------------------------------------------
# Prefix tokens (timm VisionTransformer(class_token=True, reg_tokens=R)): [cls, reg_0 .. reg_{R-1}, patches] per image
# ------------------------------------------------------------------------------------------------
def tokens_fwd(y, cls, reg, pos, B: int, N: int):
    """x0 [B * T, D] (T = N + P, P = 1 + R) from the patch rows y [B * N, D]: rows P .. T-1 of image b are y's rows of
    image b, rows 0 .. P-1 are prefix[j] (+ pos[j]) summed in fp32 and rounded once, prefix = [cls [1, D], reg [R, D]]
    (reg None when R = 0), pos [P, D] or None (prefix tokens without a position embedding)."""
    D = y.shape[1]
    pre = _f32(cls.reshape(1, D))
    if reg is not None:
        pre = torch.cat([pre, _f32(reg.reshape(-1, D))])
    if pos is not None:
        pre = pre + _f32(pos.reshape(-1, D))
    P = pre.shape[0]
    x = torch.cat([pre.to(y.dtype).expand(B, P, D), y.reshape(B, N, D)], dim=1)
    return x.reshape(B * (N + P), D)


def tokens_bwd(dx0, B: int, N: int, P: int):
    """(dpatch, dtok): the patch rows of dx0 [B * T, D] as a contiguous [B * N, D] matrix, and dtok [T, D] fp32 with
    dtok[j] = sum_b dx0[b * T + j]."""
    D = dx0.shape[1]
    x = dx0.reshape(B, N + P, D)
    return x[:, P:].reshape(B * N, D).contiguous(), x.sum(dim=0, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------
# Linear layers (timm Attention.qkv / proj, Mlp.fc1 / fc2, head) and their backward
# ------------------------------------------------------------------------------------------------
def gelu(x):
    return F.gelu(x)  # exact erf form, like timm's nn.GELU


def gelu_fwd(u):
    return F.gelu(_f32(u)).to(u.dtype)


def dgelu_mul(dg, u):
    """du = dg * gelu'(u)  (exact erf GELU)."""
    return (_f32(dg) * dgelu(u)).to(dg.dtype)


def dgelu(u):
    uf = _f32(u)
    cdf = 0.5 * (1.0 + torch.erf(uf * (1.0 / math.sqrt(2.0))))
    pdf = torch.exp(-0.5 * uf * uf) * (1.0 / math.sqrt(2.0 * math.pi))
    return cdf + uf * pdf


# ------------------------------------------------------------------------------------------------
# SwiGLU (timm SwiGLUPacked = GluMlp(act_layer=SiLU, gate_last=False)): u = [gate | value] [T, Hd], g [T, Hd / 2]
# ------------------------------------------------------------------------------------------------
def _swiglu(u):
    h = u.shape[1] // 2
    return F.silu(u[:, :h]) * u[:, h:]


def _dswiglu(dg, u):
    """du = [dg * value * silu'(gate) | dg * silu(gate)] in fp32; silu'(a) = s (1 + a (1 - s)), s = sigmoid(a)."""
    h = u.shape[1] // 2
    a, b = u[:, :h], u[:, h:]
    s = torch.sigmoid(a)
    return torch.cat([dg * b * (s * (1.0 + a * (1.0 - s))), dg * (a * s)], dim=1)


def swiglu_fwd(u):
    """g [T, Hd / 2] = silu(u[:, :Hd/2]) * u[:, Hd/2:], computed in fp32 and rounded once."""
    return _swiglu(_f32(u)).to(u.dtype)


def swiglu_bwd(dg, u):
    """du [T, Hd] = [dg * value * silu'(gate) | dg * silu(gate)], rounded to dg's dtype."""
    return _dswiglu(_f32(dg), _f32(u)).to(dg.dtype)


def linear_fwd(x, w, bias=None, act: Optional[str] = None, residual=None, res_row_mod: int = 0,
               want_preact: bool = False, ag=None, row_scale=None, rows_per_scale: int = 0):
    """y = act(x @ w.T + bias) + residual.  residual rows may be broadcast with period res_row_mod.
    row_scale (fp32 [M / rows_per_scale], no activation): y = (x @ w.T + bias) * row_scale[m / rows_per_scale]
    + residual -- the per-sample scale of stochastic depth.
    act="swiglu": w is the packed [Hd, K] fc1 weight; y = silu(u[:, :Hd/2]) * u[:, Hd/2:] [M, Hd / 2] for the
    pre-activation u = x @ w.T + bias [M, Hd] (returned as preact); no residual or row scale."""
    y = _f32(x) @ _f32(w).t()
    if bias is not None:
        y = y + _f32(bias)
    pre = y.to(x.dtype) if want_preact else None
    if act == "gelu":
        y = gelu(y)
    elif act == "swiglu":
        assert residual is None and row_scale is None, "swiglu: no residual or row scale"
        y = _swiglu(y)
    elif act is not None:
        raise ValueError(act)
    if row_scale is not None:
        assert act is None and row_scale.numel() * rows_per_scale == y.shape[0], "one scale per sample"
        y = y * row_scale.float().repeat_interleave(rows_per_scale)[:, None]
    if residual is not None:
        r = _f32(residual)
        if res_row_mod:
            reps = y.shape[0] // res_row_mod
            r = r[:res_row_mod].repeat(reps, 1)
        y = y + r
    y = y.to(x.dtype)
    return (y, pre) if want_preact else y


def linear_dgrad(dy, w, dgelu_preact=None, want_colsum: bool = False, dswiglu_preact=None):
    """dx = dy @ w  (optionally  * gelu'(preact)); colsum(dx) is the bias grad of the layer below.
    dswiglu_preact = u [M, Hd] (the packed fc1 pre-activation): dh = dy @ w is [M, Hd / 2] and the result is the fc1
    output gradient du = [dh * value * silu'(gate) | dh * silu(gate)] [M, Hd], with colsum over all Hd columns."""
    dx = _f32(dy) @ _f32(w)
    if dswiglu_preact is not None:
        dx = _dswiglu(dx, _f32(dswiglu_preact))
    elif dgelu_preact is not None:
        dx = dx * dgelu(dgelu_preact)
    dx = dx.to(dy.dtype)
    cs = _f32(dx).sum(dim=0) if want_colsum else None
    return (dx, cs) if want_colsum else dx


def linear_wgrad(dy, x, out=None):
    """dw[N, K] = dy[T, N].T @ x[T, K]"""
    dw = _f32(dy).t() @ _f32(x)
    if out is not None:
        out.copy_(dw)
        return out
    return dw.to(dy.dtype)


def colsum(x):
    return _f32(x).sum(dim=0)


# ------------------------------------------------------------------------------------------------
# Attention core (timm Attention: softmax(q k^T * hd^-0.5) v, no mask) -- run_vit_training.py:134
# qkv is the packed [T, 3*D] projection; head h of q lives at columns [h*hd, (h+1)*hd).
# ------------------------------------------------------------------------------------------------
def dropout(x, p: float, key: int):
    """y = x * keep / (1 - p); keep is a pure function of (key, position), so the checkpoint recompute and the
    backward pass regenerate it instead of storing it (reference: nn.Dropout inside timm Block / after pos_embed,
    run_vit_training.py:129,138-139)."""
    gen = torch.Generator(device=x.device)
    gen.manual_seed(int(key) & 0x7FFFFFFFFFFFFFFF)
    keep = torch.rand(x.shape, generator=gen, device=x.device) >= p
    return (x.float() * keep * (1.0 / (1.0 - p))).to(x.dtype)


# ------------------------------------------------------------------------------------------------
# Stochastic depth (timm drop_path).  The masks are bit-identical to the GPU kernels (csrc/dropout.cuh), so CPU and GPU
# runs train on the same masks and the kernels can be tested exactly against this reference.
# ------------------------------------------------------------------------------------------------
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, k0: int, k1: int):
    """Philox-4x32-10 of csrc/dropout.cuh on uint32 counter arrays (c0, c1), key (k0, k1): returns 4 uint32 arrays."""
    c0 = np.asarray(c0, dtype=np.uint64)
    c1 = np.asarray(c1, dtype=np.uint64)
    c2 = np.full_like(c0, 0x5EED5EED)
    c3 = np.full_like(c0, 0x0B200B20)
    k0, k1 = np.uint64(k0 & 0xFFFFFFFF), np.uint64(k1 & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32)
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def dropout_thresh16(p: float) -> int:
    """dropout_thresh16 of csrc/dropout.cuh, in the same fp32 arithmetic."""
    return int(np.float32(p) * np.float32(65536.0) + np.float32(0.5))


def dropout_scale(thresh16: int) -> float:
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(thresh16) / np.float32(65536.0)))


def drop_path_keep(key: int, p: float, B: int, offset: int) -> np.ndarray:
    """bool [B]: sample g = offset + b is kept iff keep bit g % 8 of dropout_keep8(g / 8, key, thresh16(p)) is set,
    i.e. iff 16-bit chunk g % 8 of Philox vector g / 8 is >= thresh16.  Keep probability 1 - thresh16 / 65536."""
    key = int(key) & 0x7FFFFFFFFFFFFFFF
    g = np.arange(offset, offset + B, dtype=np.uint64)
    i = g // np.uint64(8)
    c = (g % np.uint64(8)).astype(np.int64)
    r = np.stack(philox4x32_10(i & _M32, i >> np.uint64(32), key & 0xFFFFFFFF, key >> 32))  # [4, B]
    word = r[c >> 1, np.arange(B)].astype(np.uint32)
    chunk = (word >> ((c & 1) * 16).astype(np.uint32)) & np.uint32(0xFFFF)
    return chunk >= dropout_thresh16(p)


def drop_path_scale(key: int, p: float, B: int, offset: int, device):
    """fp32 [B]: dropout_scale(thresh16(p)) for kept samples, 0 for dropped ones."""
    keep = drop_path_keep(key, p, B, offset)
    scale = np.where(keep, np.float32(dropout_scale(dropout_thresh16(p))), np.float32(0.0)).astype(np.float32)
    return torch.from_numpy(scale).to(device)


def drop_path_bwd(dy, scale, N: int):
    """(dt = scale[row / N] * dy rounded to dy's dtype, fp32 column sums of dt)."""
    dt = (_f32(dy) * scale.float().repeat_interleave(N)[:, None]).to(dy.dtype)
    return dt, _f32(dt).sum(dim=0)


# ------------------------------------------------------------------------------------------------
# Patch dropout (timm PatchDropout(ordered=True)): the same selection bits as csrc/patch_drop.cu
# ------------------------------------------------------------------------------------------------
def patch_drop_keep(key: int, B: int, N: int, K: int, offset: int) -> np.ndarray:
    """int64 [B, K]: the patches image g = offset + b keeps, ascending.  Patch n draws r = word n % 4 of
    philox4x32_10(n / 4, g, key); the kept patches are the K smallest (r, n) pairs (a stable argsort of r)."""
    if not 1 <= K <= N:
        raise ValueError(f"patch dropout keeps 1 <= K <= N patches, got K {K}, N {N}")
    key = int(key) & 0x7FFFFFFFFFFFFFFF
    n = np.arange(N, dtype=np.uint64)
    g = np.arange(offset, offset + B, dtype=np.uint64)
    c0 = np.broadcast_to(n // np.uint64(4), (B, N))
    c1 = np.broadcast_to(g[:, None], (B, N))
    r = np.stack(philox4x32_10(c0, c1, key & 0xFFFFFFFF, key >> 32))  # [4, B, N]
    word = r[(n % np.uint64(4)).astype(np.int64)[None, :], np.arange(B)[:, None], np.arange(N)[None, :]]  # [B, N]
    order = np.argsort(word, axis=1, kind="stable")[:, :K]
    return np.sort(order, axis=1)


def patch_drop_select(key: int, B: int, N: int, K: int, offset: int, device):
    """(keep int32 [B, K], inv int32 [B, N]): keep as ``patch_drop_keep``; inv[b, n] = row of patch n in keep[b], or
    -1 when image b drops patch n."""
    keep = patch_drop_keep(key, B, N, K, offset)
    inv = np.full((B, N), -1, dtype=np.int32)
    np.put_along_axis(inv, keep, np.arange(K, dtype=np.int32)[None, :].repeat(B, 0), axis=1)
    return torch.from_numpy(keep.astype(np.int32)).to(device), torch.from_numpy(inv).to(device)


def pos_gather(pos, keep):
    """[B * K, D]: row b * K + i is pos[keep[b, i]] (the position rows of the kept patches)."""
    return pos[keep.reshape(-1).long()].contiguous()


def patch_drop_bwd(dx0, inv, B: int, N: int, K: int, P: int):
    """(dpatch, dtok) for dx0 [B * (P + K), D]: dpatch [B * K, D] = the patch rows (None when P == 0: dx0 itself is
    then the patch matrix); dtok [P + N, D] fp32, dtok[j < P] = sum_b dx0[b, j], dtok[P + n] = sum over the images that
    kept patch n of dx0[b, P + inv[b, n]], summed in b order."""
    D = dx0.shape[1]
    x = dx0.reshape(B, P + K, D)
    dtok = torch.zeros(P + N, D, dtype=torch.float32, device=dx0.device)
    dtok[:P] = x[:, :P].sum(dim=0, dtype=torch.float32)
    invl = inv.long()
    for b in range(B):
        kept = invl[b] >= 0
        dtok[P:][kept] += _f32(x[b, P:][invl[b][kept]])
    dpatch = x[:, P:].reshape(B * K, D).contiguous() if P else None
    return dpatch, dtok


def mean_pool(xn, B: int, N: int):
    """[B*N, D] -> [B, D]: mean over the tokens of an image (run_vit_training.py:161)."""
    return xn.view(B, N, -1).mean(dim=1, dtype=torch.float32).to(xn.dtype)


def mean_pool_bwd(dpooled, B: int, N: int):
    """d(mean over tokens): every token row of image b receives dpooled[b] / N."""
    D = dpooled.shape[1]
    return (dpooled.float() / N).to(dpooled.dtype)[:, None, :].expand(B, N, D).reshape(B * N, D)


def attention_fwd(qkv, B: int, N: int, H: int, hd: int, drop=None, need_p: bool = True):
    """drop = (p, key): attention dropout on the probabilities (timm Attention.attn_drop)."""
    D = H * hd
    q, k, v = _f32(qkv).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)  # [B, H, N, hd]
    s = (q @ k.transpose(-1, -2)) * (hd ** -0.5)
    p = torch.softmax(s, dim=-1).to(qkv.dtype)
    pd = p if drop is None else dropout(p, drop[0], drop[1])
    o = (_f32(pd) @ v).permute(0, 2, 1, 3).reshape(B * N, D).to(qkv.dtype)
    return o, p


# Flash-style pair: the forward keeps only the log-sum-exp of every score row, the backward rebuilds P from it
# (csrc/attention_sm90.cu on the GPU).  Off by default; tests flip FLASH_ATTENTION to exercise the model path.
FLASH_ATTENTION = False


def flash_supported(N: int, hd: int) -> bool:
    return True


def use_flash(N: int, hd: int) -> bool:
    return FLASH_ATTENTION


def _drop_scale(p, drop):
    """Mask times scale of attention dropout (p, key) for probabilities p [B, H, N, N]: the mask ``dropout`` draws for
    that shape, which is the one the un-fused path applies to its P."""
    return dropout(torch.ones_like(p, dtype=torch.float32), drop[0], drop[1])


def attention_fwd_lse(qkv, B: int, N: int, H: int, hd: int, drop=None):
    D = H * hd
    q, k, v = _f32(qkv).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * (hd ** -0.5)
    lse = torch.logsumexp(s, dim=-1)  # [B, H, N], of the undropped scores
    p = torch.exp(s - lse[..., None])
    if drop is not None:
        p = p * _drop_scale(p, drop)
    o = (p @ v).permute(0, 2, 1, 3).reshape(B * N, D).to(qkv.dtype)
    return o, lse.reshape(B * H, N).contiguous()


def attention_bwd_lse(dout, qkv, out, lse, B: int, N: int, H: int, hd: int, want_colsum: bool = False, drop=None):
    D = H * hd
    q, k, v = _f32(qkv).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    do = _f32(dout).view(B, N, H, hd).permute(0, 2, 1, 3)
    o = _f32(out).view(B, N, H, hd).permute(0, 2, 1, 3)
    p = torch.exp((q @ k.transpose(-1, -2)) * (hd ** -0.5) - lse.view(B, H, N, 1))
    delta = (do * o).sum(dim=-1, keepdim=True)  # = rowsum(dP o P) also with dropout: O is the dropped output
    ms = 1.0 if drop is None else _drop_scale(p, drop)
    dv = (p * ms).transpose(-1, -2) @ do
    ds = (hd ** -0.5) * p * ((do @ v.transpose(-1, -2)) * ms - delta)
    dq = ds @ k
    dk = ds.transpose(-1, -2) @ q
    dqkv = torch.stack([dq, dk, dv], dim=0).permute(1, 3, 0, 2, 4).reshape(B * N, 3 * D).to(qkv.dtype)
    cs = _f32(dqkv).sum(dim=0) if want_colsum else None
    return (dqkv, cs) if want_colsum else dqkv


def attention_probs(qkv, B: int, N: int, H: int, hd: int):
    """P alone (re-materialised in backward when only qkv was kept)."""
    q, k, _ = _f32(qkv).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    return torch.softmax((q @ k.transpose(-1, -2)) * (hd ** -0.5), dim=-1).to(qkv.dtype)


def attention_bwd(dout, qkv, p, B: int, N: int, H: int, hd: int, want_colsum: bool = False, drop=None):
    D = H * hd
    q, k, v = _f32(qkv).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    do = _f32(dout).view(B, N, H, hd).permute(0, 2, 1, 3)  # [B, H, N, hd]
    pf = _f32(p)
    pdrop = pf if drop is None else dropout(p, drop[0], drop[1]).float()
    dv = pdrop.transpose(-1, -2) @ do
    dp = (do @ v.transpose(-1, -2)).to(qkv.dtype)
    if drop is not None:
        dp = dropout(dp, drop[0], drop[1])  # same key, same shape -> same mask
    dp = dp.float()
    ds = (hd ** -0.5) * pf * (dp - (dp * pf).sum(dim=-1, keepdim=True))
    ds = ds.to(qkv.dtype).float()
    dq = ds @ k
    dk = ds.transpose(-1, -2) @ q
    dqkv = torch.stack([dq, dk, dv], dim=0).permute(1, 3, 0, 2, 4).reshape(B * N, 3 * D).to(qkv.dtype)
    cs = _f32(dqkv).sum(dim=0) if want_colsum else None
    return (dqkv, cs) if want_colsum else dqkv


# ------------------------------------------------------------------------------------------------
# Patch embedding (timm PatchEmbed = Conv2d(k=s=P)) as im2col + GEMM -- run_vit_training.py:124,156
# ------------------------------------------------------------------------------------------------
def mix_images(images, mix):
    """timm 0.4.12 ``Mixup._mix_batch`` (mode 'batch') in fp32 with mix = (lam, box) from ``vit.draw_mix``.
    Mixup: x * lam + x.flip(0) * (1 - lam), each product and the sum rounded to fp32 (what the fused im2col computes).
    CutMix: the box (yl, yh, xl, xh) of image b comes from image B-1-b."""
    lam, box = mix
    x = images.float()
    if box is None:
        return x * lam + x.flip(0) * (1.0 - lam)
    yl, yh, xl, xh = box
    x = x.clone()
    x[:, :, yl:yh, xl:xh] = x.flip(0)[:, :, yl:yh, xl:xh]
    return x


def patch_im2col(images, P: int, kpad: int, dtype, mix=None, keep=None):
    """keep [B, K] (patch dropout): only the kept patches, row b * K + i = patch keep[b, i] of image b."""
    if mix is not None:
        images = mix_images(images, mix)
    B, C, S, _ = images.shape
    G = S // P
    cols = images.view(B, C, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(B, G * G, C * P * P)
    if keep is not None:
        cols = torch.gather(cols, 1, keep.long()[:, :, None].expand(-1, -1, C * P * P))
    cols = cols.reshape(-1, C * P * P)
    out = torch.zeros(cols.shape[0], kpad, dtype=dtype, device=images.device)
    out[:, : C * P * P] = cols.to(dtype)
    return out


# ------------------------------------------------------------------------------------------------
# Loss (torch.nn.CrossEntropyLoss, mean) -- run_vit_training.py:229,262 ; eval argmax -- :312-313
# With mix / smoothing: timm 0.4.12 mixup_target + SoftTargetCrossEntropy (label smoothing alone is DeiT's
# LabelSmoothingCrossEntropy, i.e. F.cross_entropy(..., label_smoothing=smoothing))
# ------------------------------------------------------------------------------------------------
def mixup_target(target, num_classes: int, lam: float = 1.0, smoothing: float = 0.0):
    """timm 0.4.12 ``mixup_target``: lam * smooth(onehot(y)) + (1 - lam) * smooth(onehot(y.flip(0))), fp32."""
    off = smoothing / num_classes
    on = 1.0 - smoothing + off

    def one_hot(t):
        return torch.full((t.numel(), num_classes), off, device=t.device).scatter_(1, t.long().view(-1, 1), on)

    return one_hot(target) * lam + one_hot(target.flip(0)) * (1.0 - lam)


def cross_entropy(logits, target, want_grad: bool = True, mix=None, smoothing: float = 0.0):
    lf = _f32(logits)
    if mix is not None or smoothing > 0:
        soft = mixup_target(target, lf.shape[1], 1.0 if mix is None else mix[0], smoothing)
        logp = torch.log_softmax(lf, dim=-1)
        loss = (-soft * logp).sum(dim=-1).mean()
        dlogits = ((logp.exp() - soft) / lf.shape[0]).to(logits.dtype) if want_grad else None
        return loss, dlogits, (lf.argmax(dim=-1) == target).sum()
    lse = torch.logsumexp(lf, dim=-1)
    picked = lf.gather(1, target.view(-1, 1)).squeeze(1)
    loss = (lse - picked).mean()
    dlogits = None
    if want_grad:
        prob = torch.exp(lf - lse[:, None])
        prob[torch.arange(lf.shape[0], device=lf.device), target] -= 1.0
        dlogits = (prob / lf.shape[0]).to(logits.dtype)
    correct = (lf.argmax(dim=-1) == target).sum()
    return loss, dlogits, correct


# ------------------------------------------------------------------------------------------------
# Optimizer pieces (torch.optim.AdamW + clip_grad_norm_) -- run_vit_training.py:237,270,278
# ------------------------------------------------------------------------------------------------
def sumsq(x, out):
    out += _f32(x).pow(2).sum()


def clip_coef(sumsq_t, max_norm: float):
    norm = torch.sqrt(sumsq_t)
    return torch.clamp(max_norm / (norm + 1e-6), max=1.0), norm


def ema_update(ema, w, decay: float):
    """Model EMA step as the device computes it: ema = fmaf(d, ema, (1 - d) * w) in fp32, with d and 1 - d rounded to
    fp32.  The fused multiply-add is emulated in fp64, where the product of two fp32 values is exact; the sum is then
    rounded to fp64 and to fp32, which is one rounding more than fmaf (it can differ in the last bit on a tie)."""
    d = float(np.float32(decay))
    keep = torch.mul(w, float(np.float32(1.0) - np.float32(decay)))  # fp32 product, as on the device
    ema.copy_((ema.double() * d + keep.double()).float())


def adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step: int, ema=None, ema_decay: float = 0.0,
               groups=None, group_hyper=None):
    """ema: optional fp32 model EMA, updated from the new w (see ema_update).
    groups / group_hyper: optional parameter groups (see group_lr_decay); `wd` is then unused."""
    _adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, groups, group_hyper)
    if ema is not None:
        ema_update(ema, w, ema_decay)


def group_lr_decay(lr, groups, group_hyper, n: int):
    """Per-element (lr * lr_scale, 1 - lr * lr_scale * wd) in fp32, as the grouped kernels form them: `groups` is the
    uint8 group of every 64-element chunk, `group_hyper` the fp32 [G, 2] rows of (lr_scale, wd)."""
    if n != groups.numel() * 64:
        raise ValueError(f"grouped AdamW: {n} elements need {n // 64} chunk groups (n % 64 == 0), got {groups.numel()}")
    gh = group_hyper.to(device=groups.device, dtype=torch.float32)
    idx = groups.long().repeat_interleave(64)
    lr_e = gh[idx, 0] * torch.tensor(lr, dtype=torch.float32, device=groups.device)
    return lr_e, 1.0 - lr_e * gh[idx, 1]


def _adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step: int, groups=None, group_hyper=None):
    g = _f32(grad)
    if clip is not None:
        g = g * clip
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    denom = (v / bc2).sqrt_().add_(eps)
    if groups is None:
        w.mul_(1.0 - lr * wd)
        w.addcdiv_(m / bc1, denom, value=-lr)
    else:
        lr_e, decay = group_lr_decay(lr, groups, group_hyper, w.numel())
        w.mul_(decay)
        w.sub_(lr_e * (m / bc1) / denom)


# Split fp32 master representation: fp32 bits == (hi_bf16_bits << 16) + lo_int16, hi = nearest bf16
# (ties round up in the bit pattern so that lo always fits a signed 16-bit integer).
def split_fp32(w, hi, lo):
    bits = w.contiguous().view(torch.int32)
    rounded = bits + 0x8000  # round-half-up keeps lo within int16 for every input (ties included)
    h = rounded >> 16
    hi.copy_((h << 16).view(torch.float32).to(torch.bfloat16))
    lo.copy_((bits - (h << 16)).to(torch.int16))


def merge_fp32(hi, lo, w):
    bits = (hi.view(torch.int16).to(torch.int32) << 16) + lo.to(torch.int32)
    w.copy_(bits.view(torch.float32))


def adamw_split(hi, lo, m, v, grad, clip, lr, beta1, beta2, eps, wd, step: int, hyper=None, ema=None,
                ema_decay: float = 0.0, groups=None, group_hyper=None):
    """ema: optional (ema_hi, ema_lo), the model EMA in split form.  groups / group_hyper: as in adamw_fp32."""
    w = torch.empty(hi.shape, dtype=torch.float32, device=hi.device)
    merge_fp32(hi, lo, w)
    _adamw_fp32(w, m, v, grad, clip, lr, beta1, beta2, eps, wd, step, groups, group_hyper)
    split_fp32(w, hi, lo)
    if ema is not None:
        e = torch.empty(hi.shape, dtype=torch.float32, device=hi.device)
        merge_fp32(ema[0], ema[1], e)
        ema_update(e, w, ema_decay)
        split_fp32(e, ema[0], ema[1])
