"""The attention core against float64: the fused wgmma kernels (csrc/attention_sm90.cuh) at every tile width and
zero-padded head dim, attention dropout against a numpy Philox mask that shares no code with csrc/dropout.cuh, the
un-fused route (GEMM + row softmax kernels) and the host argument checks.

Reference.  Everything is computed in float64 from the exact bf16 inputs, sc = hd^-1/2, z = sc S with S = Q K^T:
  P = softmax(z), lse = logsumexp(z), O = (P o M s) V                        (M s: dropout mask times its scale, or 1)
  dV = (P o M s)^T dO, dP = dO V^T, delta = rowsum(dO o O_in), dS = sc P o (dP o M s - delta), dQ = dS K, dK = dS^T Q
The backward reference takes the O_in / lse_in the kernels are given: (bf16(O), fp32(lse)) of the reference, so a
forward error can neither leak into nor hide a backward error, and once the kernels' own forward outputs (the chained
test) with the bound of lse carried into the recomputed P.

Bound.  ``expected`` gives |kernel - reference| per element for every output, from float64 absolute-value products
times named constants only (u = 2^-24, u8 = 2^-8, EX2_REL, LOGF_ABS, one half bf16 ulp per stored bf16 value):
  scores        e_S = hd u (|Q| |K|^T)   (fp32 accumulation of hd exact bf16 products)
  exponent      eps = sc e_S + Z_REL (|z| + |z_max|) + EX2_REL      (Z_REL: the roundings of sc, sc log2 e, the fma
                x * sc log2 e - m * sc log2 e and of m * sc log2 e; the second term is what bites at z ~ +60)
  row sum       eps_l = sum_k P eps + (N + 2 n_tiles + 6) u      (fp32 sums; the rescale factors cancel in O / l)
  O             (P^ eps) |V| + (eps_l + u8 + (N + 2 n_tiles + 6) u) P^ |V| + half ulp   (u8: bf16 P before P V)
  lse           sc max e_S + Z_REL |z_max| + eps_l + LOGF_ABS + 6 u |ln l| + u |lse|
  backward      P from lse_in: eps_b = eps (with |lse| for |z_max|) + err(lse_in) + 2 u |lse|;  dP: e_dP = hd u |dO||V|^T;
                delta: hd u rowsum|dO o O_in|;  dS: sc P (eps_b |g| + e_dP M s + e_delta + 3 u (|dP M s| + |g|))
                + 3 u |dS| with g = dP M s - delta, then u8 |dS| (bf16 before dQ / dK);  dQ / dK / dV: the propagated
                element errors times |K| / |Q| / |dO| plus (N + 2) u of the products plus half an ulp
  un-fused      S stored as bf16 adds sc u8 (|S| + e_S) to eps; P and dP stored as bf16 add u8 relative each;
                the row softmax dot product adds N u
  column sums   against the float64 sum of the *stored* dqkv, within (rows + 64) u (sum |d| + |c0|)
FLT_MIN floors cover exp2 results that flush to zero.  The CPU meta-tests at the end show the checker accepts the
float64 result and a CPU fp32 emulation of the flash algorithm, and rejects eight specific wrong kernels at the shapes
and inputs the GPU tests use.

Inputs.  Each (image, head) slot gets one input family, so one launch covers several: scaled Gaussian scores (sc S of
std ~2.5), planted peaks (each row's maximum at key 0, N - 1, the first / last key of a 64-key tile, the last valid
key of a partial 8-key vector), a negative offset (sc S ~ -30 +- 1: a leaked zero-filled padding key, score 0, would
dominate its row), a positive offset (sc S ~ +60 +- 1), monotone rows (the row maximum grows in every key tile) and
Q = 0 (exactly uniform P).  V and dO carry a per-column mean, so |O| ~ P |V| and the bound bites.  Operands are views
into NaN-filled buffers (ld = 3D + 8 or D + 8, eight NaN rows after B N); outputs are views into sentinel canvases that
must keep their bits outside the logical region.  Every GPU test prints its worst err / tol per output (pytest -rP).
"""
import functools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_gpu_gemm_fp64 import SENTINEL, assert_untouched, poisoned, sentinel  # noqa: E402
from test_gpu_memory_bound_fp64 import FLT_MIN, U, KernelTrace, assert_within, bf16_ulp  # noqa: E402

BF16, F32 = torch.bfloat16, torch.float32
NAN = float("nan")
U8 = 2.0 ** -8             # bf16 unit roundoff
EX2_REL = 2.0 ** -21       # ex2.approx.ftz.f32 (exp2f under --use_fast_math): twice the PTX ISA bound of 2^-22
LOGF_ABS = 2.0 ** -21.41   # __logf / __log2f on [0.5, 2]; outside it 3 ulp, the 6 u |ln l| term
Z_REL = 6 * U              # roundings of sc, sc log2 e, the fma x sc log2e - m sc log2e and of m sc log2 e
KEY = 0x2545F4914F6CDD1D   # a 63-bit dropout key: both Philox key words nonzero
TILE = 64

# every head dim the fused kernels take: the 9 tile widths and the 5 zero-padded head dims
HEAD_DIMS = [32, 40, 48, 64, 72, 80, 88, 96, 104, 112, 128, 136, 144, 160]
SEQ_LENS = [2, 8, 62, 64, 66, 130, 196, 256, 576, 1024]
FAMILIES = ["gauss", "peaks", "neg", "pos", "monotone", "zero_q"]


def pad8(n):
    return (n + 7) // 8 * 8


def tile_width(hd):
    return (hd + 15) // 16 * 16


# ------------------------------------------------------------------------------------------------
# Philox4x32-10 in numpy, following the layout documented in csrc/dropout.cuh
# ------------------------------------------------------------------------------------------------
PHILOX_M = (0xD2511F53, 0xCD9E8D57)
PHILOX_W = (0x9E3779B9, 0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Random123's Philox4x32 with 10 rounds, vectorised: ctr = 4 uint32 arrays, key = 2 uint32 -> 4 uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1 = np.uint64(PHILOX_M[0]), np.uint64(PHILOX_M[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(PHILOX_W[0])) & MASK32, (k1 + np.uint64(PHILOX_W[1])) & MASK32
        p0, p1 = m0 * c[0], m1 * c[2]  # 32 x 32 -> 64-bit products, exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & MASK32]
    return [x.astype(np.uint32) for x in c]


def dropout_thresh16(p):
    """static_cast<uint32_t>(p * 65536.0f + 0.5f) with p a float."""
    return int(np.float32(np.float32(p) * np.float32(65536.0) + np.float32(0.5)))


def dropout_scale(thresh16):
    """1 / (1 - thresh16 / 65536) in float32, as the host computes it."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(thresh16) / np.float32(65536.0)))


def keep_chunks(n_vec, key):
    """The 8 16-bit chunks of Philox vectors 0 .. n_vec - 1: counter (lo32(i), hi32(i), 0x5eed5eed, 0x0b200b20), key
    (lo32(key), hi32(key)); chunk c is (r[c / 2] >> 16 (c % 2)) & 0xFFFF.  Shape [n_vec, 8], uint32."""
    i = np.arange(n_vec, dtype=np.uint64)
    n = len(i)
    r = philox4x32_10([i & MASK32, i >> np.uint64(32), np.full(n, 0x5EED5EED), np.full(n, 0x0B200B20)],
                      (key & 0xFFFFFFFF, key >> 32))
    return np.stack([(r[c >> 1] >> np.uint32(16 * (c & 1))) & np.uint32(0xFFFF) for c in range(8)], axis=1)


def attention_mask(BH, N, p, key):
    """Keep mask of the [B*H, N, pad8(N)] probability buffer cut to [B*H, N, N]: element (bh, q, k) is chunk k % 8 of
    vector (bh N + q) pad8(N) / 8 + k / 8, kept iff the chunk >= thresh16."""
    ldp = pad8(N)
    ch = keep_chunks(BH * N * ldp // 8, key).reshape(BH, N, ldp)
    return torch.from_numpy(ch[:, :, :N] >= dropout_thresh16(p))


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def peak_keys(N):
    """Keys at which the planted-peak rows put their maximum."""
    keys = [0, N - 1, min(TILE - 1, N - 1), min(TILE, N - 1), (N - 1) // TILE * TILE, N // 8 * 8 - 1 if N % 8 else N - 2]
    return sorted({k for k in keys if 0 <= k < N})


def family_qk(fam, N, hd, g):
    """(Q, K) float [N, hd] of one input family (before the bf16 rounding)."""
    # with q, k entries ~ N(0, a^2) the scaled score sc q.k has std a^2
    rn = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    if fam == "gauss":
        return rn(N, hd) * 1.6, rn(N, hd) * 1.6
    if fam == "peaks":
        K = rn(N, hd)
        keys = peak_keys(N)
        j = torch.tensor([keys[q % len(keys)] for q in range(N)])
        beta = 12.0 / math.sqrt(hd)  # sc q.k_j ~ 12 at the peak, ~N(0, beta^2) elsewhere
        return beta * K[j] + 0.05 * rn(N, hd), K
    if fam in ("neg", "pos", "monotone"):
        Q, K = rn(N, hd), rn(N, hd)  # the +-1 spread
        if fam == "monotone":
            Q, K = 0.3 * Q, 0.3 * K
            alpha = math.sqrt(20.0 * math.sqrt(hd))  # sc q.k rises from 0 to ~20 across the row
            Q[:, 0], K[:, 0] = alpha, alpha * torch.arange(N) / max(N - 1, 1)
        else:
            alpha = math.sqrt((30.0 if fam == "neg" else 60.0) * math.sqrt(hd))
            Q[:, 0], K[:, 0] = alpha, -alpha if fam == "neg" else alpha
        return Q, K
    assert fam == "zero_q"
    return torch.zeros(N, hd), rn(N, hd)


class Inputs:
    """Per-slot Q, K, V, dO [B*H, N, hd] bf16 on `device`; slot bh = b H + h gets family FAMILIES[bh % 6]."""

    def __init__(self, B, N, H, hd, device, seed=0, families=FAMILIES):
        self.B, self.N, self.H, self.hd, self.D = B, N, H, hd, H * hd
        g = torch.Generator().manual_seed(seed * 7919 + B * 1009 + N * 31 + H * 7 + hd)
        mean = torch.linspace(-2.0, 2.0, hd)  # per-column mean of V and dO
        qs, ks = zip(*[family_qk(families[bh % len(families)], N, hd, g) for bh in range(B * H)])
        self.Q = torch.stack(qs).to(BF16).to(device)
        self.K = torch.stack(ks).to(BF16).to(device)
        self.V = (torch.randn(B * H, N, hd, generator=g) + mean).to(BF16).to(device)
        self.dO = (torch.randn(B * H, N, hd, generator=g) + mean.flip(0)).to(BF16).to(device)

    def pack(self, *parts):
        """[B*H, N, hd] tensors -> [B*N, len(parts) * D] (head h of part i at columns i D + h hd)."""
        B, N, H, hd = self.B, self.N, self.H, self.hd
        return torch.stack(parts).view(len(parts), B, H, N, hd).permute(1, 3, 0, 2, 4).reshape(B * N, -1)

    def unpack(self, t, parts):
        B, N, H, hd = self.B, self.N, self.H, self.hd
        return t.reshape(B, N, parts, H, hd).permute(2, 0, 3, 1, 4).reshape(parts, B * H, N, hd)

    @functools.cached_property
    def qkv(self):
        return self.pack(self.Q, self.K, self.V)


# ------------------------------------------------------------------------------------------------
# float64 reference and the error model
# ------------------------------------------------------------------------------------------------
def half_ulp(ref, e):
    return 0.5 * bf16_ulp(ref.abs() + e)


class Forward64:
    """float64 scores, probabilities, lse and the exponent error eps of one input (route: fused or un-fused)."""

    def __init__(self, inp, Ms=None, route="fused"):
        Q, K, V = inp.Q.double(), inp.K.double(), inp.V.double()
        hd, N = inp.hd, inp.N
        self.sc = hd ** -0.5
        self.S = Q @ K.transpose(1, 2)
        self.e_S = hd * U * (Q.abs() @ K.abs().transpose(1, 2))
        self.z = self.sc * self.S
        self.lse = torch.logsumexp(self.z, -1)
        self.P = torch.exp(self.z - self.lse[..., None])
        zmax = self.z.amax(-1, keepdim=True)
        e_z = self.sc * self.e_S
        if route == "unfused":  # S stored as bf16 before the softmax kernel
            e_z = e_z + self.sc * U8 * (self.S.abs() + self.e_S)
        self.e_z = e_z
        self.eps = e_z + Z_REL * (self.z.abs() + zmax.abs()) + EX2_REL
        nt = (N + TILE - 1) // TILE
        self.c_sum = (N + 2 * nt + 6) * U
        self.eps_l = (self.P * self.eps).sum(-1, keepdim=True) + self.c_sum
        self.Ms = torch.ones_like(self.P) if Ms is None else Ms
        self.Ph = self.P * self.Ms
        self.O = self.Ph @ V
        PV = self.Ph @ V.abs()
        self.PV = PV
        floor = N * FLT_MIN * V.abs().amax((1, 2), keepdim=True)
        if route == "fused":
            e_O = (self.Ph * self.eps) @ V.abs() + (self.eps_l + U8 + self.c_sum + (U if Ms is not None else 0)) * PV
        else:  # P_bf = P (1 + eps_P); with dropout the dropout kernel rounds P s once more
            self.eps_P = self.eps + self.eps_l + (N + 2) * U + U8
            self.eps_Ph = self.eps_P + ((U + U8) if Ms is not None else 0.0)
            e_O = (self.Ph * self.eps_Ph) @ V.abs() + (N + 2) * U * PV
        self.e_O = e_O + floor + 2 * U * self.O.abs()
        l_log = torch.log(torch.exp(self.lse - zmax[..., 0]))  # ln l, l = sum exp(z - z_max) in [1, N]
        self.tol_lse = (e_z.amax(-1) + Z_REL * zmax[..., 0].abs() + self.eps_l[..., 0] + LOGF_ABS
                        + 6 * U * l_log.abs() + U * self.lse.abs())


def expected(inp, route="fused", Ms=None, out_in=None, lse_err=None, fwd=None):
    """float64 reference and bound of every output of one attention forward + backward: {name: (ref, tol)} with
    names out, lse, probs, delta, dq, dk, dv ([B*H, N, hd] / [B*H, N] / [B*H, N, N]).  route "fused" or "unfused";
    Ms the dropout mask times its scale (float64 [B*H, N, N]) or None; out_in the bf16 O the backward is given (default
    bf16 of the reference O) and lse_err the bound on its lse_in (default: fp32 rounding of the reference lse)."""
    f = fwd or Forward64(inp, Ms, route)
    N, hd, sc = inp.N, inp.hd, f.sc
    V, dO, Q, K = inp.V.double(), inp.dO.double(), inp.Q.double(), inp.K.double()
    res = {"out": (f.O, f.e_O + half_ulp(f.O, f.e_O))}
    if route == "fused":
        res["lse"] = (f.lse, f.tol_lse)
        zero_floor = FLT_MIN
        # probabilities of the second pass: exp2(x sc log2e - lse2), lse2 with the bound of lse
        eps_p = f.e_z + Z_REL * (f.z.abs() + f.lse[..., None].abs()) + EX2_REL + f.tol_lse[..., None]
        e_p = f.P * eps_p
        res["probs"] = (f.P, e_p + half_ulp(f.P, e_p) + zero_floor)
    if out_in is None:
        out_in = f.O.to(BF16)
    O_in = out_in.double()
    if lse_err is None:
        lse_err = U * f.lse.abs()
    Ms_ = f.Ms
    dP = dO @ V.transpose(1, 2)
    e_dP = hd * U * (dO.abs() @ V.abs().transpose(1, 2))
    if route == "fused":
        delta = (dO * O_in).sum(-1, keepdim=True)
        e_delta = hd * U * (dO * O_in).abs().sum(-1, keepdim=True)
        res["delta"] = (delta[..., 0], e_delta[..., 0] + U * delta[..., 0].abs())
        eps_b = (f.e_z + Z_REL * (f.z.abs() + f.lse[..., None].abs()) + EX2_REL + lse_err[..., None]
                 + 2 * U * f.lse[..., None].abs())
        g = dP * Ms_ - delta
        e_g = e_dP * Ms_ + e_delta + 3 * U * ((dP * Ms_).abs() + g.abs())
        dS = sc * f.P * g
        e_dS = sc * f.P * (eps_b * g.abs() + e_g) + 3 * U * dS.abs() + FLT_MIN * (1 + g.abs())
        eps_Ph = eps_b + U8 + 2 * U
    else:
        # dP stored as bf16; with dropout scaled and rounded again by the dropout kernel
        dpm = dP * Ms_
        e_dpm = Ms_ * (e_dP + U8 * (dP.abs() + e_dP)) + ((U + U8) * dpm.abs() if Ms is not None else 0.0)
        delta = (f.P * dpm).sum(-1, keepdim=True)  # the softmax backward's dot product: dO . O of the exact O
        e_delta = ((f.P * f.eps_P * dpm.abs() + f.P * e_dpm).sum(-1, keepdim=True)
                   + N * U * (f.P * dpm.abs()).sum(-1, keepdim=True))
        g = dpm - delta
        e_g = e_dpm + e_delta + U * g.abs()
        dS = sc * f.P * g
        e_dS = sc * f.P * (f.eps_P * g.abs() + e_g) + 4 * U * dS.abs() + FLT_MIN * (1 + g.abs())
        eps_b = None
        eps_Ph = f.eps_Ph
    e_dS = e_dS + U8 * (dS.abs() + e_dS)  # bf16 dS before the dQ / dK products
    dQ, dK = dS @ K, dS.transpose(1, 2) @ Q
    e_dQ = e_dS @ K.abs() + (N + 2) * U * (dS.abs() @ K.abs())
    e_dK = e_dS.transpose(1, 2) @ Q.abs() + (N + 2) * U * (dS.abs().transpose(1, 2) @ Q.abs())
    Ph = f.Ph
    dV = Ph.transpose(1, 2) @ dO
    e_dV = ((Ph * eps_Ph + FLT_MIN).transpose(1, 2) @ dO.abs()
            + (N + 2) * U * (Ph.transpose(1, 2) @ dO.abs()))
    for name, ref, e in (("dq", dQ, e_dQ), ("dk", dK, e_dK), ("dv", dV, e_dV)):
        res[name] = (ref, e + half_ulp(ref, e))
    if route == "unfused":
        res["probs"] = (f.P, f.P * f.eps_P + FLT_MIN)
    return res


def expected_softmax_fwd(S, sc, n):
    """Row softmax of bf16 scores S [rows, n] (float64 reference, bound)."""
    z = sc * S.double()
    zmax = z.amax(-1, keepdim=True)
    P = torch.softmax(z, -1)
    eps = Z_REL * (z.abs() + zmax.abs()) + EX2_REL
    e = P * (eps + (P * eps).sum(-1, keepdim=True) + (n + 2) * U)
    return P, e + half_ulp(P, e) + FLT_MIN


def expected_softmax_bwd(P, dP, sc, n):
    """dS = sc P (dP - rowsum(P dP)) of bf16 P, dP [rows, n] (float64 reference, bound)."""
    P, dP = P.double(), dP.double()
    dot = (P * dP).sum(-1, keepdim=True)
    e_dot = n * U * (P * dP).abs().sum(-1, keepdim=True)
    g = dP - dot
    dS = sc * P * g
    e = sc * P.abs() * (e_dot + U * g.abs()) + 4 * U * dS.abs()
    return dS, e + half_ulp(dS, e)


# ------------------------------------------------------------------------------------------------
# checking
# ------------------------------------------------------------------------------------------------
class Margins:
    """|got - ref| <= tol per element, with the worst err / tol ratio kept per output and reported."""

    def __init__(self):
        self.worst = {}

    def check(self, name, got, ref, tol):
        ref, tol = ref.to(got.device), tol.to(got.device)
        err = (got.double() - ref).abs()
        ratio = torch.nan_to_num(err / tol.clamp_min(1e-300), nan=math.inf)
        r = float(ratio.max()) if ratio.numel() else 0.0
        key = name.split(":")[-1].strip()
        self.worst[key] = max(self.worst.get(key, 0.0), r)
        try:
            assert_within(name, got, ref, tol)
        except AssertionError as e:
            raise AssertionError(f"{e}; worst err / tol {r:.3g}") from None

    def colsum(self, name, cs, c0, d, rows):
        """Column sums that started at c0, against c0 + the float64 sum of the stored bf16 values d (over dim 0)."""
        d64 = d.double()
        self.check(name, cs, c0 + d64.sum(0), (rows + 64) * U * (d64.abs().sum(0) + abs(c0)))

    def report(self):
        print("worst err / tol: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items())))


class Flat:
    """A contiguous `shape` view at the start of a sentinel-filled flat buffer with 64 spare elements."""

    def __init__(self, shape, dtype, device, fill=None):
        n = math.prod(shape)
        self.buf = sentinel((n + 64,), dtype, device)
        self.view = self.buf[:n].view(shape)
        if fill is not None:
            self.view.fill_(fill)

    def untouched(self, name, written=None):
        mask = torch.zeros(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        mask[:self.view.numel()] = True if written is None else written.flatten()
        assert_untouched(name, self.buf, mask)


def device_kernels(trace):
    """Names of the kernels a stopped KernelTrace recorded on the device."""
    from torch.autograd import DeviceType

    return sorted({e.name for e in trace.prof.events() if e.device_type == DeviceType.CUDA})


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _C():
    return _co()._C


# ------------------------------------------------------------------------------------------------
# fused kernels: one forward (with lse and probs, and without either) + one backward, checked
# ------------------------------------------------------------------------------------------------
def run_fused(m, inp, case, drop=None, chained=False, probs=True):
    """Runs the fused kernels on poisoned operands into sentinel canvases and checks every output against float64."""
    C = _C()
    B, N, H, hd, D = inp.B, inp.N, inp.H, inp.hd, inp.D
    BH, dev = B * H, inp.Q.device
    p, key = drop if drop is not None else (0.0, 0)
    Ms = None
    if drop is not None:
        Ms = attention_mask(BH, N, p, key).to(dev).double() * dropout_scale(dropout_thresh16(p))
    route = "fused"
    fwd = Forward64(inp, Ms, route)
    qkv, _ = poisoned(inp.qkv)
    # forward with lse (and the probabilities without dropout)
    out = Flat((B * N, D), BF16, dev)
    lse = Flat((BH, N), F32, dev)
    ldp = pad8(N) + 8
    pr = Flat((BH, N, ldp), BF16, dev) if (probs and drop is None) else None
    C.attention_fwd(qkv, out.view, lse.view, pr.view if pr is not None else None, B, N, H, hd, float(p), key)
    # the same forward without lse / probabilities: bitwise the same O
    out2 = Flat((B * N, D), BF16, dev)
    C.attention_fwd(qkv, out2.view, None, None, B, N, H, hd, float(p), key)
    # backward from the reference (O, lse), or from the kernels' own (chained)
    if chained:
        o_in, lse_in = out.view.clone(), lse.view.clone()
    else:
        o_in, lse_in = inp.pack(fwd.O.to(BF16)), fwd.lse.to(F32)
    exp = expected(inp, route, Ms, out_in=inp.unpack(o_in, 1)[0],
                   lse_err=fwd.tol_lse if chained else None, fwd=fwd)
    dout_v, _ = poisoned(inp.pack(inp.dO))
    o_in_v, _ = poisoned(o_in)
    lse_in_v = Flat((BH, N), F32, dev)
    lse_in_v.view.copy_(lse_in)
    delta = Flat((BH, N), F32, dev)
    dqkv = Flat((B * N, 3 * D), BF16, dev)
    c0 = 0.25
    cs = Flat((3 * D,), F32, dev, fill=c0)
    C.attention_bwd(qkv, dout_v, o_in_v, lse_in_v.view, delta.view, dqkv.view, cs.view, B, N, H, hd, float(p), key)

    got_out = inp.unpack(out.view, 1)[0]
    m.check(f"{case}: out", got_out, *exp["out"])
    assert torch.equal(out.view.view(torch.int16), out2.view.view(torch.int16)), f"{case}: out differs without lse"
    m.check(f"{case}: lse", lse.view, *exp["lse"])
    if pr is not None:
        m.check(f"{case}: probs", pr.view[:, :, :N], *exp["probs"])
        written = torch.zeros(pr.view.shape, dtype=torch.bool, device=dev)
        written[:, :, :N] = True
        pr.untouched(f"{case}: probs canvas", written)
    m.check(f"{case}: delta", delta.view, *exp["delta"])
    dq, dk, dv = inp.unpack(dqkv.view, 3)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        m.check(f"{case}: {name}", got, *exp[name])
    m.colsum(f"{case}: colsum", cs.view, c0, dqkv.view, B * N)
    for name, fl in (("out", out), ("out (no lse)", out2), ("lse", lse), ("delta", delta), ("dqkv", dqkv),
                     ("colsum", cs)):
        fl.untouched(f"{case}: {name} canvas")


def fused_names(hd, drop=False):
    w = tile_width(hd)
    if drop:
        return [f"attn_fwd_drop_sm90_kernel<{w}>", f"attn_bwd_drop_sm90_kernel<{w}, 0>",
                f"attn_bwd_drop_sm90_kernel<{w}, 1>"]
    return [f"attn_fwd_sm90_kernel<{w}>", f"attn_bwd_sm90_kernel<{w}, 0>", f"attn_bwd_sm90_kernel<{w}, 1>",
            "attn_delta_kernel"]


# every head dim at N in {66, 196, 576}, every N at hd in {40, 64, 160}; (B, H) with 6 slots, one per family
FUSED_CASES = sorted({(hd, N) for hd in HEAD_DIMS for N in (66, 196, 576)} |
                     {(hd, N) for hd in (40, 64, 160) for N in SEQ_LENS})


@pytest.mark.gpu
@pytest.mark.parametrize("hd,N", FUSED_CASES, ids=[f"hd{hd}-N{N}" for hd, N in FUSED_CASES])
def test_fused_against_fp64(hd, N):
    inp = Inputs(2, N, 3, hd, "cuda")
    m = Margins()
    trace = KernelTrace()
    try:
        run_fused(m, inp, f"hd {hd} N {N}")
        for k in fused_names(hd):
            trace.expect(k)
        trace.verify()
    finally:
        trace.stop()
    m.report()


@pytest.mark.gpu
def test_fused_grid_larger_than_resident():
    """B = 3, H = 16, N = 576: 432 work items, more than 132 SMs hold at once."""
    inp = Inputs(3, 576, 16, 64, "cuda")
    m = Margins()
    run_fused(m, inp, "B3 H16 N576 hd64")
    m.report()


@pytest.mark.gpu
@pytest.mark.parametrize("hd,N", [(64, 196), (72, 130), (160, 576), (40, 1024)])
def test_fused_chained_forward_backward(hd, N):
    """The backward fed the kernels' own forward outputs; the bound of lse is carried into the recomputed P."""
    inp = Inputs(2, N, 3, hd, "cuda", seed=1)
    m = Margins()
    run_fused(m, inp, f"chained hd {hd} N {N}", chained=True, probs=False)
    m.report()


# ------------------------------------------------------------------------------------------------
# attention dropout against the numpy Philox mask
# ------------------------------------------------------------------------------------------------
DROP_HEAD_DIMS = [32, 40, 64, 72, 88, 104, 128, 136, 160]  # one per tile width: 32 48 64 80 96 112 128 144 160
DROP_P = [0.1, 0.5, 2.0 ** -18]  # the last rounds to thresh16 = 0: everything kept, s = 1


@pytest.mark.gpu
@pytest.mark.parametrize("p", DROP_P, ids=["p0.1", "p0.5", "p2^-18"])
@pytest.mark.parametrize("hd", DROP_HEAD_DIMS)
def test_fused_dropout_against_fp64(hd, p):
    N = 196 if hd % 3 else 66  # N % 8 != 0: the last Philox vector of every row is partial
    inp = Inputs(2, N, 3, hd, "cuda", seed=2)
    m = Margins()
    trace = KernelTrace()
    try:
        run_fused(m, inp, f"hd {hd} N {N} p {p:g}", drop=(p, KEY))
        for k in fused_names(hd, drop=True):
            trace.expect(k)
        trace.verify()
    finally:
        trace.stop()
    m.report()


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.1, 0.5, 2.0 ** -18])
def test_standalone_dropout_matches_numpy_philox(p):
    """co.dropout bitwise: y = bf16(x s) where the numpy mask keeps, +0 where it drops."""
    co = _co()
    BH, N = 6, 197
    ldp = pad8(N)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(BH, N, ldp, generator=g).to(BF16).cuda()
    y = co.dropout(x, p, KEY)
    keep = torch.from_numpy(keep_chunks(BH * N * ldp // 8, KEY).reshape(BH, N, ldp) >= dropout_thresh16(p)).cuda()
    want = torch.where(keep, (x.float() * dropout_scale(dropout_thresh16(p))).to(BF16), torch.zeros_like(x))
    bad = y.view(torch.int16) != want.view(torch.int16)
    assert not bool(bad.any()), f"{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


# ------------------------------------------------------------------------------------------------
# the un-fused route: row softmax kernels, and attention_fwd / attention_bwd end to end
# ------------------------------------------------------------------------------------------------
# n -> the instance softmax_fwd / softmax_bwd dispatch to
SOFTMAX_ROUTES = {2: "softmax_{}_kernel<2>", 128: "softmax_{}_kernel<2>", 256: "softmax_{}_kernel<4>",
                  576: "softmax_{}_kernel<9>", 578: "softmax_{}_kernel<16>", 1024: "softmax_{}_kernel<16>",
                  1: "softmax_{}_vec_kernel<1>", 49: "softmax_{}_vec_kernel<1>", 257: "softmax_{}_vec_kernel<2>",
                  1023: "softmax_{}_vec_kernel<4>", 1025: "softmax_{}_vec_kernel<8>",
                  2049: "softmax_{}_long_kernel", 4096: "softmax_{}_long_kernel"}


def softmax_rows(n, g):
    """Score rows [13, n] (13: a partial block of 8 rows): offset (-30 and +60 sc-units), peaked (max at the first,
    the last and the last-but-one column, and one in the middle), Gaussian."""
    sc = 64 ** -0.5
    rows = []
    for r in range(13):
        kind = r % 4
        x = torch.randn(n, generator=g)
        if kind == 0:
            x = (-30.0 + x) / sc
        elif kind == 1:
            x = (60.0 + x) / sc
        elif kind == 2:
            x = 2.5 * x / sc
            x[[0, n - 1, max(n - 2, 0), n // 2][r // 4 % 4]] = 14.0 / sc
        else:
            x = 2.5 * x / sc
        rows.append(x)
    return torch.stack(rows).to(BF16), sc


@pytest.mark.gpu
@pytest.mark.parametrize("n", list(SOFTMAX_ROUTES))
def test_softmax_kernels_against_fp64(n):
    C = _C()
    g = torch.Generator().manual_seed(n)
    S, sc = softmax_rows(n, g)
    rows, ld = S.shape[0], pad8(n) + 8
    m = Margins()
    trace = KernelTrace()
    try:
        buf = torch.full((rows, ld), NAN, dtype=BF16, device="cuda")
        buf[:, :n] = S.cuda()
        pad = buf[:, n:].clone()
        C.softmax_fwd(buf, rows, n, ld, sc)
        m.check(f"n {n}: softmax fwd", buf[:, :n], *expected_softmax_fwd(S.cuda(), sc, n))
        assert torch.equal(buf[:, n:].view(torch.int16), pad.view(torch.int16)), f"n {n}: fwd wrote padding"
        P = buf[:, :n].clone()
        dP = (torch.randn(rows, n, generator=g) + 1.0).to(BF16).cuda()
        dbuf = torch.full((rows, ld), NAN, dtype=BF16, device="cuda")
        dbuf[:, :n] = dP
        C.softmax_bwd(dbuf, buf, rows, n, ld, sc)
        m.check(f"n {n}: softmax bwd", dbuf[:, :n], *expected_softmax_bwd(P, dP, sc, n))
        assert torch.equal(dbuf[:, n:].view(torch.int16), pad.view(torch.int16)), f"n {n}: bwd wrote padding"
        for d in ("fwd", "bwd"):
            trace.expect(SOFTMAX_ROUTES[n].format(d))
        trace.verify()
    finally:
        trace.stop()
    m.report()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 49])
def test_softmax_zero_rows_is_a_noop(n):
    """rows = 0 launches nothing and raises nothing, on the pair (even n) and the vector (odd n) route."""
    C = _C()
    ld = pad8(n) + 8
    buf = sentinel((4, ld), BF16, "cuda")
    p = sentinel((4, ld), BF16, "cuda")
    trace = KernelTrace()
    try:
        C.softmax_fwd(buf, 0, n, ld, 0.125)
        C.softmax_bwd(buf, p, 0, n, ld, 0.125)
    finally:
        trace.stop()
    assert not device_kernels(trace), device_kernels(trace)
    assert bool((buf.view(torch.int16) == SENTINEL[BF16]).all())


UNFUSED_CASES = ([(N, 56) for N in (1, 49, 197, 577)] + [(N, 80) for N in (1, 49, 197, 577)]
                 + [(197, 120), (577, 152), (49, 152), (1, 120)])


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [False, True], ids=["plain", "dropout"])
@pytest.mark.parametrize("N,hd", UNFUSED_CASES, ids=[f"N{N}-hd{hd}" for N, hd in UNFUSED_CASES])
def test_unfused_route_against_fp64(N, hd, drop):
    """cuda_ops.attention_fwd / attention_bwd at odd N, at head dims no fused kernel takes and at hd = 80, which the
    default routing sends un-fused."""
    co = _co()
    inp = Inputs(1, N, 6, hd, "cuda", seed=3)
    B, H, D = inp.B, inp.H, inp.D
    p = 0.1
    Ms = None
    if drop:
        Ms = attention_mask(B * H, N, p, KEY).cuda().double() * dropout_scale(dropout_thresh16(p))
    exp = expected(inp, "unfused", Ms)
    m = Margins()
    qkv, _ = poisoned(inp.qkv)
    dout, _ = poisoned(inp.pack(inp.dO))
    trace = KernelTrace()
    try:
        out, P = co.attention_fwd(qkv, B, N, H, hd, drop=(p, KEY) if drop else None)
        dqkv, cs = co.attention_bwd(dout, qkv, P, B, N, H, hd, want_colsum=True, drop=(p, KEY) if drop else None)
        trace.expect("softmax_fwd", absent=("attn_",))
        trace.expect("softmax_bwd")
        trace.verify()
    finally:
        trace.stop()
    case = f"N {N} hd {hd}{' dropout' if drop else ''}"
    m.check(f"{case}: out", inp.unpack(out, 1)[0], *exp["out"])
    m.check(f"{case}: probs", P[:, :, :N], *exp["probs"])
    dq, dk, dv = inp.unpack(dqkv, 3)
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        m.check(f"{case}: {name}", got, *exp[name])
    m.colsum(f"{case}: colsum", cs, 0.0, dqkv, B * N)
    m.report()


# ------------------------------------------------------------------------------------------------
# host checks: every bad argument raises before anything is launched
# ------------------------------------------------------------------------------------------------
def _bad_calls():
    """(name, fwd or bwd, argument overrides) for B = 1, N = 64, H = 2, hd = 64."""
    B, N, H, hd = 1, 64, 2, 64
    D, dev = H * hd, "cuda"
    bf = lambda *s: torch.zeros(*s, dtype=BF16, device=dev)  # noqa: E731
    f32 = lambda *s: torch.zeros(*s, dtype=F32, device=dev)  # noqa: E731
    base_fwd = dict(qkv=bf(B * N, 3 * D), out=bf(B * N, D), lse=f32(B * H, N), probs=None, B=B, N=N, H=H, hd=hd,
                    drop_p=0.0, drop_key=0)
    base_bwd = dict(qkv=bf(B * N, 3 * D), dout=bf(B * N, D), out=bf(B * N, D), lse=f32(B * H, N),
                    delta=f32(B * H, N), dqkv=bf(B * N, 3 * D), colsum=None, B=B, N=N, H=H, hd=hd, drop_p=0.0,
                    drop_key=0)
    wide = lambda r, c, extra: bf(r, c + extra)[:, :c]  # noqa: E731  row stride c + extra
    big_bf, big_f = bf(B * N * 3 * D + 8), f32(B * H * N + 8)
    cases = [
        ("fwd qkv odd row stride", "fwd", dict(qkv=wide(B * N, 3 * D, 1))),
        ("fwd qkv row stride not a multiple of 8", "fwd", dict(qkv=wide(B * N, 3 * D, 4))),
        ("fwd qkv base not 16-byte aligned", "fwd", dict(qkv=big_bf[4:4 + B * N * 3 * D].view(B * N, 3 * D))),
        ("fwd qkv short", "fwd", dict(qkv=bf(B * N - 1, 3 * D))),
        ("fwd qkv narrow", "fwd", dict(qkv=bf(B * N, 3 * D - 8))),
        ("fwd out short", "fwd", dict(out=bf(B * N - 2, D))),
        ("fwd out strided", "fwd", dict(out=wide(B * N, D, 8))),
        ("fwd out misaligned", "fwd", dict(out=big_bf[1:1 + B * N * D].view(B * N, D))),
        ("fwd lse short", "fwd", dict(lse=f32(B * H, N - 1))),
        ("fwd lse bf16", "fwd", dict(lse=bf(B * H, N))),
        ("fwd probs ldp < N", "fwd", dict(probs=bf(B * H, N, N - 8))),
        ("fwd probs odd ldp", "fwd", dict(N=62, qkv=bf(B * 62, 3 * D), out=bf(B * 62, D), lse=f32(B * H, 62),
                                          probs=bf(B * H, 62, 63))),
        ("fwd probs wrong rows", "fwd", dict(probs=bf(B * H - 1, N, N))),
        ("fwd probs misaligned", "fwd", dict(probs=bf(B * H * N * N + 1)[1:].view(B * H, N, N))),
        ("fwd probs with dropout", "fwd", dict(probs=bf(B * H, N, N), drop_p=0.1)),
        ("fwd odd N", "fwd", dict(N=63, qkv=bf(B * 63, 3 * D), out=bf(B * 63, D), lse=f32(B * H, 63))),
        ("fwd head dim 56", "fwd", dict(hd=56, H=2, qkv=bf(B * N, 3 * 112), out=bf(B * N, 112))),
        ("fwd dropout p >= 1", "fwd", dict(drop_p=1.0)),
        ("bwd qkv odd row stride", "bwd", dict(qkv=wide(B * N, 3 * D, 1))),
        ("bwd qkv short", "bwd", dict(qkv=bf(B * N - 1, 3 * D))),
        ("bwd qkv narrow", "bwd", dict(qkv=bf(B * N, 3 * D - 8))),
        ("bwd dout odd row stride", "bwd", dict(dout=wide(B * N, D, 1))),
        ("bwd dout base not 16-byte aligned", "bwd", dict(dout=big_bf[2:2 + B * N * D].view(B * N, D))),
        ("bwd dout short", "bwd", dict(dout=bf(B * N - 1, D))),
        ("bwd out odd row stride", "bwd", dict(out=wide(B * N, D, 1))),
        ("bwd out base not 4-byte aligned", "bwd", dict(out=big_bf[1:1 + B * N * D].view(B * N, D))),
        ("bwd out narrow", "bwd", dict(out=bf(B * N, D - 8))),
        ("bwd lse base not 8-byte aligned", "bwd", dict(lse=big_f[1:1 + B * H * N].view(B * H, N))),
        ("bwd delta base not 8-byte aligned", "bwd", dict(delta=big_f[1:1 + B * H * N].view(B * H, N))),
        ("bwd lse short", "bwd", dict(lse=f32(B * H, N - 2))),
        ("bwd dqkv short", "bwd", dict(dqkv=bf(B * N - 1, 3 * D))),
        ("bwd dqkv strided", "bwd", dict(dqkv=wide(B * N, 3 * D, 8))),
        ("bwd dqkv misaligned", "bwd", dict(dqkv=big_bf[1:1 + B * N * 3 * D].view(B * N, 3 * D))),
        ("bwd colsum short", "bwd", dict(colsum=f32(3 * D - 1))),
        ("bwd dropout p < 0", "bwd", dict(drop_p=-0.1)),
        ("bwd head dim 56", "bwd", dict(hd=56)),
    ]
    return base_fwd, base_bwd, cases


@pytest.mark.gpu
def test_host_rejects_bad_arguments():
    """Each bad argument alone: a RuntimeError, and no kernel at all ran (the delta kernel included)."""
    C = _C()
    base_fwd, base_bwd, cases = _bad_calls()
    torch.cuda.synchronize()
    for name, which, over in cases:
        kw = dict(base_fwd if which == "fwd" else base_bwd, **over)
        fn = C.attention_fwd if which == "fwd" else C.attention_bwd
        trace = KernelTrace()
        try:
            with pytest.raises(RuntimeError):
                fn(**kw)
        finally:
            trace.stop()
        names = device_kernels(trace)
        assert not names, f"{name}: kernels ran before the error: {names}"
    # the unchanged base arguments are accepted
    C.attention_fwd(**base_fwd)
    C.attention_bwd(**base_bwd)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# CPU: Philox known answers, and the checker against correct and wrong emulated kernels
# ------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10 (the generic core, any counter words 2 and 3)."""
    vectors = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
               ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
               ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
                (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in vectors:
        got = philox4x32_10([np.array([c]) for c in ctr], key)
        assert tuple(int(x[0]) for x in got) == want, (ctr, key, [hex(int(x[0])) for x in got])


def test_dropout_threshold_and_scale():
    assert dropout_thresh16(2.0 ** -18) == 0 and dropout_scale(0) == 1.0
    assert dropout_thresh16(0.5) == 32768 and dropout_scale(32768) == 2.0
    t = dropout_thresh16(0.1)
    assert t == 6554 and abs(dropout_scale(t) - 1 / (1 - 6554 / 65536)) < 1e-6


def flash_emulated(inp, sc=None, Ms=None, leak=False, drop_last=False, l_dropped=False):
    """The fused forward's arithmetic in fp32 on the CPU: 64-key tiles, online max / rescale, bf16-rounded unnormalised
    P before P V, final bf16 store.  Mutants: one zero padding key leaked in, the last valid key masked out, another
    scale, l summed over the dropped probabilities.  Returns (out [B*H, N, hd] bf16, lse fp32)."""
    q, k, v = inp.Q.float(), inp.K.float(), inp.V.float()
    BH, N = q.shape[:2]
    sc = inp.hd ** -0.5 if sc is None else sc
    ms = torch.ones(BH, N, N) if Ms is None else Ms.float()
    if leak:  # a zero-filled key / value row past N takes part in the softmax
        k, v = torch.cat([k, torch.zeros(BH, 1, inp.hd)], 1), torch.cat([v, torch.zeros(BH, 1, inp.hd)], 1)
        ms = torch.cat([ms, torch.ones(BH, N, 1)], 2)
    if drop_last:
        k, v, ms = k[:, :-1], v[:, :-1], ms[:, :, :-1]
    sl2 = float(np.float32(np.float32(sc) * np.float32(1.4426950408889634)))
    S = q @ k.transpose(1, 2)
    nk = S.shape[2]
    m = torch.full((BH, N), -math.inf)
    lsum = torch.zeros(BH, N)
    o = torch.zeros(BH, N, inp.hd)
    for t in range(0, nk, TILE):
        x = S[:, :, t:t + TILE]
        mn = torch.maximum(m, x.amax(-1))
        f = torch.exp2((m - mn) * sl2)
        pt = torch.exp2(x * sl2 - (mn * sl2)[..., None])
        pm = pt * ms[:, :, t:t + TILE]
        lsum = lsum * f + (pm if l_dropped else pt).sum(-1)
        o = o * f[..., None] + pm.to(BF16).float() @ v[:, t:t + TILE]
        m = mn
    return (o / lsum[..., None]).to(BF16), m * sc + torch.log(lsum)


def bwd_emulated(inp, out_in, lse_in, Ms=None, ds_mask_after=False, transposed_kv=False):
    """The fused backward in fp32 on the CPU (P from lse, dS rounded to bf16, bf16 stores).  Mutants: dS = sc P o (dP
    - delta) o M s, and the mask transposed in the dK / dV role.  Returns (dq, dk, dv) [B*H, N, hd] bf16."""
    q, k, v, do = inp.Q.float(), inp.K.float(), inp.V.float(), inp.dO.float()
    BH, N = q.shape[:2]
    sc = inp.hd ** -0.5
    ms = torch.ones(BH, N, N) if Ms is None else Ms.float()
    P = torch.exp2((q @ k.transpose(1, 2)) * (sc * 1.4426950408889634) - (lse_in * 1.4426950408889634)[..., None])
    dP = do @ v.transpose(1, 2)
    delta = (do * out_in.float()).sum(-1, keepdim=True)

    def ds(mask):
        if ds_mask_after:
            return (sc * P * (dP - delta) * mask).to(BF16).float()
        return (sc * P * (dP * mask - delta)).to(BF16).float()

    mk = ms.transpose(1, 2) if transposed_kv else ms
    dq = ds(ms) @ k
    dk = ds(mk).transpose(1, 2) @ q
    dv = (P * mk).to(BF16).float().transpose(1, 2) @ do
    return dq.to(BF16), dk.to(BF16), dv.to(BF16)


META_SHAPES = [(72, 196), (136, 66), (40, 130), (64, 2), (160, 256)]


def _meta_inputs(hd, N):
    return Inputs(2, N, 3, hd, "cpu")


def _mask(inp, p):
    return attention_mask(inp.B * inp.H, inp.N, p, KEY).double() * dropout_scale(dropout_thresh16(p))


@pytest.mark.parametrize("hd,N", META_SHAPES)
@pytest.mark.parametrize("p", [None, 0.1], ids=["plain", "dropout"])
def test_checker_accepts_fp64_and_emulated_flash(hd, N, p):
    inp = _meta_inputs(hd, N)
    Ms = _mask(inp, p) if p else None
    exp = expected(inp, "fused", Ms)
    m = Margins()
    ref_o, ref_lse = exp["out"][0], exp["lse"][0]
    m.check("fp64: out", ref_o.to(BF16), *exp["out"])
    m.check("fp64: lse", ref_lse.float(), *exp["lse"])
    m.check("fp64: probs", exp["probs"][0].to(BF16), *exp["probs"])
    o, lse = flash_emulated(inp, Ms=Ms)
    m.check("fp32 flash: out", o, *exp["out"])
    m.check("fp32 flash: lse", lse, *exp["lse"])
    grads = bwd_emulated(inp, ref_o.to(BF16), ref_lse.float(), Ms)
    for name, got in zip(("dq", "dk", "dv"), grads):
        m.check(f"fp64: {name}", exp[name][0].to(BF16), *exp[name])
        m.check(f"fp32 flash: {name}", got, *exp[name])
    # the chained bound accepts the emulated backward fed the emulated forward
    chained = expected(inp, "fused", Ms, out_in=o, lse_err=exp["lse"][1])
    for name, got in zip(("dq", "dk", "dv"), bwd_emulated(inp, o, lse, Ms)):
        m.check(f"chained: {name}", got, *chained[name])
    m.report()


@pytest.mark.parametrize("hd,N", [(56, 49), (80, 197), (152, 1)])
def test_checker_accepts_unfused_emulation(hd, N):
    """The un-fused route's roundings in fp32 on the CPU: S, P, dP and dS stored as bf16."""
    inp = Inputs(1, N, 6, hd, "cpu", seed=3)
    Ms = _mask(inp, 0.1)
    exp = expected(inp, "unfused", Ms)
    q, k, v, do = inp.Q.float(), inp.K.float(), inp.V.float(), inp.dO.float()
    sc = hd ** -0.5
    S = (q @ k.transpose(1, 2)).to(BF16).float()
    P = torch.softmax(S * sc, -1).to(BF16).float()
    Ph = (P * Ms.float()).to(BF16).float()
    m = Margins()
    m.check("out", (Ph @ v).to(BF16), *exp["out"])
    m.check("probs", P, *exp["probs"])
    dpm = ((do @ v.transpose(1, 2)).to(BF16).float() * Ms.float()).to(BF16).float()
    dS = (sc * P * (dpm - (P * dpm).sum(-1, keepdim=True))).to(BF16).float()
    for name, got in (("dq", dS @ k), ("dk", dS.transpose(1, 2) @ q), ("dv", Ph.transpose(1, 2) @ do)):
        m.check(name, got.to(BF16), *exp[name])
    m.report()


def _rejects(name, got, ref, tol):
    with pytest.raises(AssertionError, match="worst err / tol"):
        Margins().check(name, got, ref, tol)


@pytest.mark.parametrize("hd,N", [(72, 196), (136, 66), (40, 130)])
def test_checker_rejects_mask_mutants(hd, N):
    """1. a zero-filled padding key leaked into the softmax; 2. the last valid key masked out (N % 64 != 0)."""
    inp = _meta_inputs(hd, N)
    exp = expected(inp, "fused")
    o, lse = flash_emulated(inp, leak=True)
    _rejects("leaked key: out", o, *exp["out"])
    _rejects("leaked key: lse", lse, *exp["lse"])
    o, lse = flash_emulated(inp, drop_last=True)
    _rejects("last key dropped: out", o, *exp["out"])


@pytest.mark.parametrize("hd", [72, 136])
def test_checker_rejects_tile_width_scale(hd):
    """3. sc taken from the tile width instead of hd."""
    inp = _meta_inputs(hd, 196)
    exp = expected(inp, "fused")
    o, lse = flash_emulated(inp, sc=tile_width(hd) ** -0.5)
    _rejects("tile-width scale: out", o, *exp["out"])
    _rejects("tile-width scale: lse", lse, *exp["lse"])


@pytest.mark.parametrize("hd,N", [(72, 196), (160, 66)])
def test_checker_rejects_dropout_mutants(hd, N):
    """4. l summed over the dropped probabilities; 5. dS = sc P o (dP - delta) o M s; 6. the mask transposed in the
    dK / dV role."""
    inp = _meta_inputs(hd, N)
    Ms = _mask(inp, 0.1)
    exp = expected(inp, "fused", Ms)
    o, lse = flash_emulated(inp, Ms=Ms, l_dropped=True)
    _rejects("l over dropped P: out", o, *exp["out"])
    _rejects("l over dropped P: lse", lse, *exp["lse"])
    o_in, lse_in = exp["out"][0].to(BF16), exp["lse"][0].float()
    dq, dk, _ = bwd_emulated(inp, o_in, lse_in, Ms, ds_mask_after=True)
    _rejects("mask after delta: dq", dq, *exp["dq"])
    _rejects("mask after delta: dk", dk, *exp["dk"])
    _, dk, dv = bwd_emulated(inp, o_in, lse_in, Ms, transposed_kv=True)
    _rejects("transposed mask: dv", dv, *exp["dv"])
    _rejects("transposed mask: dk", dk, *exp["dk"])


@pytest.mark.parametrize("hd,N", [(64, 196), (40, 130)])
def test_checker_rejects_colsum_skipping_last_tile(hd, N):
    """7. the column sums skip the rows of the last partial tile."""
    inp = _meta_inputs(hd, N)
    exp = expected(inp, "fused")
    d = inp.pack(*(exp[k][0].to(BF16) for k in ("dq", "dk", "dv")))
    full = torch.cat([torch.arange(b * N, b * N + N // TILE * TILE) for b in range(inp.B)])
    with pytest.raises(AssertionError, match="worst err / tol"):
        Margins().colsum("colsum", 0.25 + d[full].double().sum(0).float(), 0.25, d, inp.B * N)


@pytest.mark.parametrize("n", [2, 128, 578, 1024])
def test_checker_rejects_softmax_missing_last_pair(n):
    """8. the pair kernel skips the last pair of a row: it takes no part in max / sum and keeps its input."""
    g = torch.Generator().manual_seed(n)
    S, sc = softmax_rows(n, g)
    P, tol = expected_softmax_fwd(S, sc, n)
    got = S.clone()
    if n > 2:
        got[:, :n - 2] = torch.softmax(sc * S[:, :n - 2].float(), -1).to(BF16)
    _rejects("softmax missing last pair", got, P, tol)
    # and the correct fp32 softmax passes
    Margins().check("softmax fp32", torch.softmax(sc * S.float(), -1).to(BF16), P, tol)
