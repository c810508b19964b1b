"""Memory-bound sm_90a kernels (csrc/elementwise.cu, csrc/layernorm_stream.cu) against float64 references.

Every reference below is computed from the same bf16 / fp32 tensors the kernel reads, upcast to float64, and is
checked against ``torch.autograd`` / ``torch.optim`` in the CPU meta-tests at the end of the file.  The tolerances are
derived from the arithmetic the kernels do (written next to each checker), in units of u = 2^-24 (fp32 unit roundoff)
and of one bf16 ulp of the float64 value; the meta-tests show each checker accepts the exact reference and rejects
specific wrong kernels.

Every LayerNorm case (and the fused-epilogue GELU case) also asserts, from a torch.profiler trace, which kernel
instances ran: the dispatch picks among a dozen template instances by width, row count and environment, and a matrix
that silently drifts onto another route tests nothing it claims to.

Run as a script (``python tests/test_gpu_memory_bound_fp64.py small|register``) it checks the LayerNorm routes that
only ``B200_LN_SMALL=0`` / ``B200_LN_STREAM=0`` select; the extension reads those once per process.
"""
import math
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from vit_10b_fsdp_example_b200.models.vit import BLOCK_LN_EPS, FINAL_LN_EPS  # noqa: E402

U = 2.0 ** -24  # fp32 unit roundoff
FLT_MIN = 2.0 ** -126


def _f32(v: float) -> float:
    """A host scalar as the kernel receives it (a float argument)."""
    return float(np.float32(v))


# ------------------------------------------------------------------------------------------------
# checking helpers
# ------------------------------------------------------------------------------------------------
def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at each float64 value: 2^(e - 8) for |ref| = m 2^e, m in [0.5, 1); 2^-133 below FLT_MIN."""
    _, e = torch.frexp(ref.abs().clamp_min(FLT_MIN))
    return torch.ldexp(torch.ones_like(ref), e - 8)


def assert_within(name, got, ref, tol):
    """|got - ref| <= tol element-wise (NaN fails); the message names the worst element."""
    got64 = got.double()
    err = (got64 - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        ratio = torch.where(bad, err / tol.clamp_min(1e-300), torch.zeros_like(err))
        i = int(torch.argmax(torch.nan_to_num(ratio, nan=math.inf)).item())
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements outside tolerance; worst at flat "
                             f"index {i}: got {got64.flatten()[i].item()!r}, ref {ref.flatten()[i].item()!r}, "
                             f"tol {tol.flatten()[i].item()!r}")


class KernelTrace:
    """Names of the CUDA kernels launched between construction and verify() (torch.profiler, CUDA activities),
    checked against the kernels the test expects: a substring of the demangled name, e.g. 'ln_bwd_kernel<4>'.
    One session spans a whole test and is padded with idle time on both sides: short per-launch sessions late in a
    long process came back without their kernel records."""

    PAD_S = 0.1

    def __init__(self):
        from torch.profiler import ProfilerActivity, profile

        self.want, self.avoid, self.running = [], [], True
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.start()
        time.sleep(self.PAD_S)

    def expect(self, kernel, absent=()):
        self.want.append(kernel)
        self.avoid.extend(absent)

    def stop(self):
        if self.running:
            torch.cuda.synchronize()
            time.sleep(self.PAD_S)
            self.prof.stop()
            self.running = False

    def verify(self):
        self.stop()
        names = sorted({e.name for e in self.prof.events()})
        for k in self.want:
            assert any(k in n for n in names), f"expected a launch of {k}; trace: {names}"
        for a in self.avoid:
            assert not any(a in n for n in names), f"unexpected launch of {a}; trace: {names}"


@pytest.fixture
def trace():
    t = KernelTrace()
    yield t
    t.stop()


def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------
# LayerNorm: float64 references and checkers
# ------------------------------------------------------------------------------------------------
def ln_fwd_ref(x, g, b, eps, ddof=0):
    """y, mean, rstd, std in float64 (ddof=1 is a mutant for the meta-tests: variance over D - 1)."""
    x64 = x.double()
    mean = x64.mean(1)
    var = (x64 - mean[:, None]).square().sum(1) / (x.shape[1] - ddof)
    rstd = (var + eps).rsqrt()
    y = (x64 - mean[:, None]) * rstd[:, None] * g.double() + b.double()
    return y, mean, rstd, var.sqrt()


def ln_bwd_ref(dy, x, g, mean, rstd, dres=None):
    """dx, dgamma, dbeta in float64 at the given statistics (not recomputed: the backward is judged on its own)."""
    x64, dy64, g64 = x.double(), dy.double(), g.double()
    mean64, rstd64 = mean.double()[:, None], rstd.double()[:, None]
    xhat = (x64 - mean64) * rstd64
    gdy = g64 * dy64
    dx = rstd64 * (gdy - gdy.mean(1, keepdim=True) - xhat * (gdy * xhat).mean(1, keepdim=True))
    if dres is not None:
        dx = dx + dres.double()
    return dx, (dy64 * xhat).sum(0), dy64.sum(0)


def check_ln_fwd(x, g, b, eps, y, mean, rstd):
    """y: one bf16 ulp plus an fp32 floor.  The kernel sums a row in fp32 (a serial sum of at most 32 elements per
    thread, then a tree of at most 8 levels), so |mean error| <= 64 u mean_j|x_j|; that error reaches y through
    (x - mean) rstd g.  rsqrt.approx and the fp32 products add a few u of |g xhat| and |b|:
        |y - y64| <= ulp(y64) + 64 u (|g| rstd mean_j|x_j| + |g xhat|) + 4 u |b|
    mean and rstd: relative 1e-5 against (|mean| + std) and against rstd."""
    y64, mean64, rstd64, std64 = ln_fwd_ref(x, g, b, eps)
    x64, g64 = x.double(), g.double()
    xhat = (x64 - mean64[:, None]) * rstd64[:, None]
    floor = 64 * U * (g64.abs() * (rstd64 * x64.abs().mean(1))[:, None] + (g64 * xhat).abs()) + 4 * U * b.double().abs()
    assert_within("ln_fwd y", y, y64, bf16_ulp(y64) + floor)
    assert_within("ln_fwd mean", mean, mean64, 1e-5 * (mean64.abs() + std64))
    assert_within("ln_fwd rstd", rstd, rstd64, 1e-5 * rstd64)


def check_ln_bwd(dy, x, g, mean, rstd, dres, dx, dgamma, dbeta, dxsum):
    """dx: one bf16 ulp plus an fp32 floor.  The row sums m1 = mean(g dy) and m2 = mean(g dy xhat) carry at most
    64 u of mean|g dy| and mean|g dy xhat| (same summation shape as the forward); the wide-row stream kernel folds dx
    into dres + rstd g dy - k1 x + k0 with k1 = rstd m2 rstd, k0 = k1 mean - rstd m1, whose cancellation costs
    u |k1| (|x| + |mean|); the remaining products and sums a few u of each term:
        |dx - dx64| <= ulp(dx64) + 64 u rstd (mean|g dy| + (|xhat| + rstd (|x| + |mean|)) mean|g dy xhat|)
                       + 4 u (rstd |g dy| + |dres|)
    dgamma, dbeta: relative 1e-5 of sum_rows |dy xhat| and sum_rows |dy| per column.
    dxsum: the column sums of the dx the kernel returned (bf16), i.e. the bias gradient a GEMM colsum would give,
    to 1e-6 sum_rows |dx|; summing the fp32 values before rounding is off by ~2^-9 0.4 / sqrt(rows) of that."""
    dx64, dg64, db64 = ln_bwd_ref(dy, x, g, mean, rstd, dres)
    x64, dy64, g64 = x.double(), dy.double(), g.double()
    mean64, rstd64 = mean.double()[:, None], rstd.double()[:, None]
    xhat = (x64 - mean64) * rstd64
    gdy = g64 * dy64
    a1, a2 = gdy.abs().mean(1, keepdim=True), (gdy * xhat).abs().mean(1, keepdim=True)
    floor = 64 * U * rstd64 * (a1 + (xhat.abs() + rstd64 * (x64.abs() + mean64.abs())) * a2)
    floor = floor + 4 * U * (rstd64 * gdy.abs() + (dres.double().abs() if dres is not None else 0))
    assert_within("ln_bwd dx", dx, dx64, bf16_ulp(dx64) + floor)
    assert_within("ln_bwd dgamma", dgamma, dg64, 1e-5 * (dy64 * xhat).abs().sum(0))
    assert_within("ln_bwd dbeta", dbeta, db64, 1e-5 * dy64.abs().sum(0))
    if dxsum is not None:
        dxk = dx.double()
        assert_within("ln_bwd dxsum", dxsum, dxk.sum(0), 1e-6 * dxk.abs().sum(0))


def ln_inputs(rows, D, seed, device):
    """bf16 x, gamma, beta, dy, dres.  Rows cycle through: |mean| >> std (64 + N(0, 1), quantised to bf16 at a 0.5
    step), N(0, 1), a constant row (var = 0: rstd = eps^-1/2, y = beta), N(0.5, 2).  Every 7th gamma is zero."""
    gen = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(rows, D, generator=gen, device=device)
    kind = torch.arange(rows, device=device) % 4
    x[kind == 0] += 64.0
    const = (torch.randn(rows, 1, generator=gen, device=device) * 2).expand(rows, D)
    x = torch.where((kind == 2)[:, None], const, x)
    x = torch.where((kind == 3)[:, None], x * 2 + 0.5, x)
    g = torch.randn(D, generator=gen, device=device)
    g[::7] = 0
    b = torch.randn(D, generator=gen, device=device)
    dy = torch.randn(rows, D, generator=gen, device=device)
    dres = torch.randn(rows, D, generator=gen, device=device)
    return tuple(t.to(torch.bfloat16) for t in (x, g, b, dy, dres))


def _tpr(D):
    nv = D // 8
    return 32 if nv <= 32 else 64 if nv <= 64 else 128 if nv <= 128 else 256


def ln_fwd_kernel_name(D, small=True):
    """csrc/elementwise.cu layernorm_fwd: rows of D <= 2048 share a CTA (TPR threads each) unless B200_LN_SMALL=0;
    wider rows take one CTA each with ceil(D / 2048) 16-byte vectors per thread."""
    if D <= 2048 and small:
        return f"ln_fwd_small_kernel<{_tpr(D)}>"
    return f"ln_fwd_kernel<{(D // 8 + 255) // 256}>"


def ln_bwd_kernel_name(D, rows, res, dxsum, sm, small=True, stream=True):
    """csrc/elementwise.cu layernorm_bwd: small kernel as in the forward; the bulk-copy stream kernel for whole
    512-column multiples when there is at least one row per SM (384-thread build up to D = 5632, else 672), unless
    B200_LN_STREAM=0; otherwise the register-resident wide kernel."""
    if D <= 2048 and small:
        return f"ln_bwd_small_kernel<{_tpr(D)}>"
    if stream and D >= 2048 and D % 512 == 0 and D // 16 <= 640 and rows >= sm:
        return f"ln_bwd_stream_kernel<{str(res).lower()}, {str(dxsum).lower()}, {384 if 32 + D // 16 <= 384 else 672}>"
    return f"ln_bwd_kernel<{(D // 8 + 255) // 256}>"


LN_WIDTHS = [8, 192, 384, 1024, 1152, 1280, 1408, 1664, 1792, 2048, 2056, 2304, 2560, 4096, 5120, 6144, 8192]
LN_ROWS = ["one", "ragged", "few", "strided", "ring"]


def ln_rows(kind, D, sm):
    if D <= 2048:
        per_cta = 256 // _tpr(D)
        stride = 6 * sm * per_cta  # the forward grid (6 CTAs / SM) is the larger of the two small-kernel grids
    else:
        per_cta, stride = 1, 8 * sm  # one row per CTA; forward grid 8 CTAs / SM, backward at most 3
    return {
        "one": 1,
        "ragged": 37 * per_cta + per_cta // 2 + 1,  # not a multiple of the rows per CTA
        "few": sm - 5,                              # fewer rows than SMs: register wide backward
        "strided": stride + 3,                      # the grid-stride loops run twice for some CTAs
        "ring": 3 * sm + 7,                         # not a multiple of the stream kernel's grid (one CTA per SM)
    }[kind]


def run_ln_case(trace, D, rows, seed, small=True, stream=True):
    """Forward at both model eps values, then the backward for every (dres, dxsum) combination, at the float64
    statistics rounded to fp32; every launch is routed to the kernel the dispatch promises."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    sm = sm_count()
    x, g, b, dy, dres = ln_inputs(rows, D, seed, "cuda")
    for eps in (BLOCK_LN_EPS, FINAL_LN_EPS):
        y, mean, rstd = co.ln_fwd(x, g, b, eps)
        trace.expect(ln_fwd_kernel_name(D, small))
        check_ln_fwd(x, g, b, _f32(eps), y, mean, rstd)
    _, mean64, rstd64, _ = ln_fwd_ref(x, g, b, _f32(FINAL_LN_EPS))
    mean, rstd = mean64.float(), rstd64.float()
    for res in (False, True):
        for want in (False, True):
            r = dres if res else None
            dx, dg, db, dxs = co.ln_bwd(dy, x, g, mean, rstd, dres=r, want_dxsum=want)
            trace.expect(ln_bwd_kernel_name(D, rows, res, want, sm, small, stream))
            assert (dxs is not None) == want
            check_ln_bwd(dy, x, g, mean, rstd, r, dx, dg, db, dxs)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", LN_ROWS)
@pytest.mark.parametrize("D", LN_WIDTHS)
def test_layernorm_matrix(D, kind, trace):
    run_ln_case(trace, D, ln_rows(kind, D, sm_count()), seed=D * 10 + LN_ROWS.index(kind))
    trace.verify()


# Widths the forced routes run: with B200_LN_SMALL=0 the narrow rows take ln_fwd_kernel<1> / ln_bwd_kernel<1>; with
# B200_LN_STREAM=0 the stream-eligible widths take the register wide backward.
FORCED = {
    "small": ("B200_LN_SMALL", [(8, "ragged"), (1024, "strided"), (2048, "ring")]),
    "register": ("B200_LN_STREAM", [(2560, "ring"), (5120, "strided"), (6144, "ring"), (8192, "ring")]),
}


def _forced_main(which):
    torch.cuda.set_device(0)
    sm = sm_count()
    for D, kind in FORCED[which][1]:
        trace = KernelTrace()
        run_ln_case(trace, D, ln_rows(kind, D, sm), seed=D, small=which != "small", stream=which != "register")
        trace.verify()
        print(f"ok {which} D={D} rows={ln_rows(kind, D, sm)}")


@pytest.mark.gpu
@pytest.mark.parametrize("which", sorted(FORCED))
def test_layernorm_forced_routes(which):
    env = dict(os.environ)
    env[FORCED[which][0]] = "0"
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), which], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert p.stdout.count("ok ") == len(FORCED[which][1]), p.stdout


# ------------------------------------------------------------------------------------------------
# GELU / dGELU on every finite bf16 input
# ------------------------------------------------------------------------------------------------
def finite_bf16_grid():
    """All 65,536 bf16 bit patterns except NaN and +-inf (exponent field all ones), as a [256, 256] grid with the
    256 excluded slots set to zero.  Infinities are left out on purpose: the erf polynomial gives NaN for -inf
    (-inf * (1 + erf) = -inf * 0)."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(torch.bfloat16)
    finite = ((bits.int() >> 7) & 0xFF) != 0xFF
    return torch.where(finite, v, torch.zeros_like(v)).reshape(256, 256), int(finite.sum())


def gelu_ref(x):
    x64 = x.double()
    return 0.5 * x64 * torch.special.erfc(-x64 / math.sqrt(2.0))  # erfc: no cancellation in 1 + erf for x << 0


def dgelu_ref(x):
    x64 = x.double()
    return 0.5 * torch.special.erfc(-x64 / math.sqrt(2.0)) + x64 * torch.exp(-0.5 * x64 * x64) / math.sqrt(2 * math.pi)


def _ftz(x, ref):
    """The build uses --use_fast_math (fp32 subnormals flush to zero): where |x| or |ref| is below 2^-125 the
    result may be a flushed 0, so the whole |ref| is allowed there."""
    tiny = (x.double().abs() < 2.0 ** -125) | (ref.abs() < 2.0 ** -125)
    return torch.where(tiny, ref.abs(), torch.zeros_like(ref))


ERF_TOL = 2e-7  # GELU approximation term, per unit |x| (gelu) or per unit |dg| (1 + |x|) (dgelu): see the checkers


def check_gelu(x, got):
    """One bf16 ulp, plus |x| 2e-7: the Abramowitz-Stegun erf (elementwise.cu erf_poly, gemm_sm90.cu erf_as) is
    within 1.5e-7 and 1 + erf is formed in fp32, so 0.5 x (1 + erf) carries up to |x| (0.75e-7 + u) more."""
    ref = gelu_ref(x)
    assert_within("gelu", got, ref, bf16_ulp(ref) + x.double().abs() * ERF_TOL + _ftz(x, ref))


def check_dgelu(x, dg, got):
    """dg * gelu'(x): one bf16 ulp, plus |dg| (1 + |x|) 2e-7 -- the erf error enters the cdf term (0.75e-7, not
    scaled by x) and the fp32 x pdf product carries a few u of |x| pdf."""
    ref = dg.double() * dgelu_ref(x)
    assert_within("dgelu", got, ref, bf16_ulp(ref) + dg.double().abs() * (1 + x.double().abs()) * ERF_TOL)


@pytest.mark.gpu
def test_gelu_every_bf16_standalone():
    """gelu_fwd / dgelu_mul: the routes ViT-L/H/g/G/e take (K < FUSE_ACT_MIN_K), with dg = 1 and a random dg."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    grid, n = finite_bf16_grid()
    assert n == 65536 - 256
    u = grid.cuda()
    g = co.gelu_fwd(u)
    check_gelu(u, g)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for dg in (torch.ones_like(u), torch.randn(u.shape, generator=gen, device="cuda").to(torch.bfloat16)):
        du = co.dgelu_mul(dg, u)
        check_dgelu(u, dg, du)


@pytest.mark.gpu
def test_gelu_every_bf16_fused_epilogue(trace):
    """The GEMM epilogue's GELU and dGELU on the same inputs.  The pre-activations are exact: A = I (one-hot rows)
    times B = grid^T puts exactly one bf16 product, grid[m, n] * 1, in every accumulator; for the dgrad, A = diag(dg)
    times an all-ones B gives acc[m, n] = dg[m] exactly, multiplied by gelu'(aux_in[m, n])."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    grid, _ = finite_bf16_grid()
    u = grid.cuda()
    n = 256
    eye = torch.eye(n, device="cuda", dtype=torch.bfloat16)
    bt = u.t().contiguous()
    out = torch.empty(n, n, device="cuda", dtype=torch.bfloat16)
    co.gemm_raw(eye, n, 0, bt, n, 0, out, n, n, n, n, act=co.ACT_GELU)
    trace.expect("gemm_bf16_sm90_kernel", absent=("gelu_fwd_kernel",))
    check_gelu(u, out)
    gen = torch.Generator(device="cuda").manual_seed(2)
    ones = torch.ones(n, n, device="cuda", dtype=torch.bfloat16)
    for dgr in (torch.ones(n, device="cuda"), torch.randn(n, generator=gen, device="cuda")):
        dgr = dgr.to(torch.bfloat16)
        a = torch.diag(dgr)
        d = torch.empty(n, n, device="cuda", dtype=torch.bfloat16)
        co.gemm_raw(a, n, 0, ones, n, 0, d, n, n, n, n, aux_in=u, ld_aux=n, act=co.ACT_DGELU)
        trace.expect("gemm_bf16_sm90_kernel", absent=("dgelu_mul_kernel",))
        check_dgelu(u, dgr[:, None].expand(n, n), d)
    trace.verify()


# ------------------------------------------------------------------------------------------------
# cross entropy (hard, smoothed, mixed)
# ------------------------------------------------------------------------------------------------
def ce_ref(logits, target, lam=1.0, smoothing=0.0, last_tie=False):
    """loss, dlogits, per-row lse and target weights t, correct -- float64.  t = off + (on - off)(lam [c == y_b] +
    (1 - lam) [c == y_{B-1-b}]) (timm mixup_target).  last_tie=True is a mutant: argmax takes the last tie."""
    z = logits.double()
    B, C = z.shape
    off = smoothing / C
    on = 1.0 - smoothing + off
    t = torch.full_like(z, off)
    rows = torch.arange(B, device=z.device)
    t[rows, target] += (on - off) * lam
    if lam != 1.0:
        t[rows, target.flip(0)] += (on - off) * (1.0 - lam)
    lse = torch.logsumexp(z, 1)
    loss = (lse - (t * z).sum(1)).mean()
    dl = (torch.softmax(z, 1) - t) / B
    arg = (C - 1 - z.flip(1).argmax(1)) if last_tie else z.argmax(1)  # torch.argmax: first index on ties
    return loss, dl, lse, t, int((arg == target).sum())


def check_ce(logits, target, lam, smoothing, loss, dl, correct):
    """Per row the kernel forms lse - picked in fp32: lse = max + log(sum exp) with the exp terms summed over a
    256-thread stride (at most C / 256 serial adds, 8 tree levels) and ex2 / lg2.approx, the smoothing term sums the
    C logits the same way, and the rows meet in fp32 atomics:
        row error <= (C / 256 + 16) u (|lse| + sum_c |t_c z_c|) + (C / 256 + 32) u,  loss error <= mean of those
                     + B u mean|row loss|
    dlogits = bf16((exp(z - lse) - t) / B): one bf16 ulp plus p (lse error + 2^-20 + 2 u |z - lse|) / B + 2 u t / B,
    and a flushed 0 below 2^-125 (--use_fast_math).
    correct: exact (first index wins a tied maximum, as torch.argmax)."""
    loss64, dl64, lse, t, correct64 = ce_ref(logits, target, lam, smoothing)
    B, C = logits.shape
    z = logits.double()
    row_err = (C / 256 + 16) * U * (lse.abs() + (t * z).abs().sum(1)) + (C / 256 + 32) * U
    row_loss = (lse - (t * z).sum(1)).abs()
    tol = row_err.mean() + B * U * row_loss.mean()
    assert_within("cross_entropy loss", loss.reshape(()), loss64, tol)
    if dl is not None:
        p = torch.softmax(z, 1)
        dtol = (p * (row_err[:, None] + 2.0 ** -20 + 2 * U * (z - lse[:, None]).abs()) + 2 * U * t) / B
        assert_within("cross_entropy dlogits", dl, dl64, bf16_ulp(dl64) + dtol + _ftz(dl64, dl64))
    assert int(correct) == correct64, f"correct {int(correct)} != {correct64}"


def ce_inputs(B, C, seed, device):
    """Logits N(0, 20^2) clipped to +-60, bf16.  Every third row has its maximum twice (at j1 < j2); the target sits
    on the first copy in two of every three of those rows and on the second in the third (an even split would let a
    last-index argmax keep the same count)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    z = (torch.randn(B, C, generator=gen, device=device) * 20).clamp(-60, 60)
    target = torch.randint(0, C, (B,), generator=gen, device=device)
    for b in range(0, B, 3):
        j1, j2 = (b * 7) % (C - 1), C - 1 - (b % 3)
        j1, j2 = min(j1, j2), max(j1, j2)
        if j1 == j2:
            j1 = j2 - 1
        z[b, j1] = z[b, j2] = 61.0
        target[b] = j2 if (b // 3) % 3 == 2 else j1
    return z.to(torch.bfloat16), target


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 128, 257])
@pytest.mark.parametrize("C", [10, 1000, 1001, 21843])
def test_cross_entropy(C, B):
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    logits, target = ce_inputs(B, C, seed=C + B, device="cuda")
    modes = [(1.0, 0.0), (1.0, 0.1)] + ([(0.3, 0.1), (0.7, 0.0)] if B % 2 == 0 else [])
    for lam, sm in modes:
        mix = None if lam == 1.0 else (lam, None)
        loss, dl, correct = co.cross_entropy(logits, target, mix=mix, smoothing=sm)
        check_ce(logits, target, lam, sm, loss, dl, correct)
        loss_ng, dl_ng, correct_ng = co.cross_entropy(logits, target, want_grad=False, mix=mix, smoothing=sm)
        assert dl_ng is None
        # the rows meet in fp32 atomics whose order is not fixed, so two runs agree to the reordering bound only
        # (bit-identical for B = 1, 3 on H100; not for B = 128, 257)
        _, _, lse, t, _ = ce_ref(logits, target, lam, sm)
        row_loss = (lse - (t * logits.double()).sum(1)).abs()
        assert abs(loss_ng.item() - loss.item()) <= 2 * B * U * float(row_loss.mean()), (loss_ng.item(), loss.item())
        assert int(correct_ng) == int(correct)


# ------------------------------------------------------------------------------------------------
# mean pool, colsum, sumsq, clip_coef
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 1280, 1408, 5120])
@pytest.mark.parametrize("N", [1, 3, 196, 257, 1369])
def test_mean_pool(N, D):
    """Forward: the kernel sums the N tokens serially in fp32 (4 loads in flight, then the n + 4 > N tail) and
    multiplies by 1/N: |pooled - mean| <= ulp + (N + 3) u mean_n|x|.  Backward: bf16(dp / N) to one bf16 ulp."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    B = 3
    gen = torch.Generator(device="cuda").manual_seed(N * 7 + D)
    xn = (torch.randn(B * N, D, generator=gen, device="cuda") + 0.5).to(torch.bfloat16)
    pooled = co.mean_pool(xn, B, N)
    x64 = xn.double().view(B, N, D)
    ref = x64.mean(1)
    assert_within("meanpool_fwd", pooled, ref, bf16_ulp(ref) + (N + 3) * U * x64.abs().mean(1))
    dp = torch.randn(B, D, generator=gen, device="cuda").to(torch.bfloat16)
    dxn = co.mean_pool_bwd(dp, B, N)
    dref = (dp.double() / N)[:, None, :].expand(B, N, D).reshape(B * N, D)
    assert_within("meanpool_bwd", dxn, dref, bf16_ulp(dref))


def _colsum64(x, chunk=8192):
    s = torch.zeros(x.shape[1], dtype=torch.float64, device=x.device)
    a = torch.zeros_like(s)
    for r in range(0, x.shape[0], chunk):
        blk = x[r:r + chunk].double()
        s += blk.sum(0)
        a += blk.abs().sum(0)
    return s, a


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [1, 5, 100003])
@pytest.mark.parametrize("C", [8, 2056, 15360])
def test_colsum(C, rows):
    """The kernel sums a slab of rows_per rows serially per column, then adds the slab sums with fp32 atomics:
    |colsum - sum| <= (rows_per + slabs) u sum_r|x| (slabs and rows_per as colsum() in elementwise.cu picks them).
    At C = 15360 the row count is capped at 16411 (500 MB of bf16) to keep the test small on a shared GPU."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    rows = min(rows, 16411) if C == 15360 else rows
    gen = torch.Generator(device="cuda").manual_seed(C + rows)
    x = torch.randn(rows, C, generator=gen, device="cuda", dtype=torch.bfloat16) + 0.25
    out = co.colsum(x)
    gx = (C // 8 + 255) // 256
    slabs = max(1, sm_count() * 4 // gx)
    rows_per = max(1, -(-rows // slabs))
    slabs = -(-rows // rows_per)
    ref, mag = _colsum64(x)
    assert_within("colsum", out, ref, (rows_per + slabs) * U * mag)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 255, 257, 2 ** 24 + 3])
def test_sumsq(n, dtype):
    """Each thread sums its grid-stride elements serially, a CTA adds its 256 partials in a tree (8 levels) and the
    CTAs meet in one fp32 atomic: all terms are positive, so |sumsq - ref| <= (per_thread + 8 + grid) u ref."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    gen = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, generator=gen, device="cuda").to(dtype)
    out = torch.zeros(1, device="cuda")
    co.sumsq(x, out)
    ref = x.double().square().sum().reshape(1)
    grid = min(-(-n // 256), sm_count() * 8)
    per_thread = -(-n // (grid * 256))
    assert_within("sumsq", out, ref, (per_thread + 8 + grid) * U * ref)


def clip_ref(sumsq, max_norm):
    """torch clip_grad_norm_: norm = sqrt(sum of squares), coef = min(1, max_norm / (norm + 1e-6))."""
    norm = math.sqrt(sumsq)
    return min(1.0, max_norm / (norm + _f32(1e-6))), norm


@pytest.mark.gpu
@pytest.mark.parametrize("max_norm", [1.0, 0.37])
def test_clip_coef(max_norm):
    """sqrt.approx (2 u), div.approx (2 u) and the +1e-6: within 16 u relative."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    mn = _f32(max_norm)
    for s in (0.0, _f32((0.5 * mn) ** 2), _f32(mn * mn), _f32((3 * mn) ** 2), _f32(1e6)):
        t = torch.tensor([s], device="cuda")
        coef, norm = co.clip_coef(t, mn)
        cref, nref = clip_ref(s, mn)
        assert_within(f"clip_coef({s})", coef, torch.tensor([cref], dtype=torch.float64, device="cuda"),
                      torch.full((1,), 16 * U * cref, dtype=torch.float64, device="cuda"))
        assert_within(f"norm({s})", norm, torch.tensor([nref], dtype=torch.float64, device="cuda"),
                      torch.full((1,), 16 * U * nref, dtype=torch.float64, device="cuda"))
        if s == 0.0:
            assert coef.item() == 1.0


# ------------------------------------------------------------------------------------------------
# AdamW
# ------------------------------------------------------------------------------------------------
def adamw_ref(w, m, v, g, coef, lr, b1, b2, eps, wd, step):
    """One torch.optim.AdamW step (decoupled decay, then the bias-corrected Adam update) in float64."""
    w, m, v, g = w.double(), m.double(), v.double(), g.double() * coef
    w = w * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    upd = (lr / bc1) * m / (v.sqrt() / math.sqrt(bc2) + eps)
    return w - upd, m, v, upd


def check_adamw(w0, m0, v0, g, coef, hp, step, w, m, v):
    """From the same fp32 state: m and v are fp32 products and a sum (3 u and 6 u of their terms); the new w is an
    fp32 product with the decay, the update (approximate divides and sqrt, the bias corrections: within 32 u of the
    update formed from |b1 m0| + |(1 - b1) g|, since m itself may cancel) and a difference:
        |w - w64| <= 2 u (|w0| + |w64|) + 32 u (lr / bc1) (b1 |m0| + (1 - b1) |g|) / (sqrt(v64 / bc2) + eps)"""
    lr, b1, b2, eps, wd = hp
    w64, m64, v64, _ = adamw_ref(w0, m0, v0, g, coef, lr, b1, b2, eps, wd, step)
    gc = g.double().abs() * coef
    upd = (lr / (1 - b1 ** step)) * (b1 * m0.double().abs() + (1 - b1) * gc) / (
        v64.sqrt() / math.sqrt(1 - b2 ** step) + eps)
    assert_within("adamw m", m, m64, 3 * U * (b1 * m0.double().abs() + (1 - b1) * gc))
    assert_within("adamw v", v, v64, 6 * U * (b2 * v0.double() + (1 - b2) * gc * gc))
    assert_within("adamw w", w, w64, 2 * U * (w0.double().abs() + w64.abs()) + 32 * U * upd.abs())


def check_split(hi, lo, merged):
    """The split master: (hi, lo) is exactly split_fp32 of the merged fp32 value, and hi is the nearest bf16 with
    ties rounding away from zero."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    hi2, lo2 = torch.empty_like(hi), torch.empty_like(lo)
    co.split_fp32(merged, hi2, lo2)
    assert torch.equal(hi2.view(torch.int16), hi.view(torch.int16)) and torch.equal(lo2, lo)
    w64, h64 = merged.double(), hi.double()
    half = bf16_ulp(w64) / 2
    d = (w64 - h64).abs()
    assert bool((d <= half).all()), "hi is not the nearest bf16"
    tie = d == half
    assert bool((h64[tie].abs() > w64[tie].abs()).all()), "a tie did not round away from zero"


def adamw_state(n, step, seed):
    """w of both signs: N(0, 0.02), a quarter tiny (+-1e-5, they cross zero in one step), and every 16th an exact
    bf16 tie (low 16 bits 0x8000); zero moments at step 1, else moments of a run in progress."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn(n, generator=gen, device="cuda") * 0.02
    w[::4] = torch.randn(w[::4].shape, generator=gen, device="cuda") * 1e-5
    wi = w.view(torch.int32)
    wi[::16] = (wi[::16] & ~0xFFFF) | 0x8000
    if step == 1:
        m, v = torch.zeros_like(w), torch.zeros_like(w)
    else:
        m = torch.randn(n, generator=gen, device="cuda") * 1e-3
        v = (torch.randn(n, generator=gen, device="cuda") * 1e-3).square()
    return w, m, v


ADAM_STEPS = [1, 2, 10, 1000, 10000]


@pytest.mark.gpu
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("flavour", ["split", "split_hyper", "fp32"])
def test_adamw(flavour, gdtype, clip):
    """adamw_split with the host step, adamw_split with the device hyper block [lr, step] (what the training loop
    passes: the host lr / step are then wrong on purpose and must be ignored), and adamw_fp32; n % 4 in 0..3 (the
    4-wide body and the scalar tail), at the bias corrections of steps 1, 2, 10, 1000 and 10000."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    hp = tuple(_f32(t) for t in (1e-3, 0.9, 0.999, 1e-8, 0.1))
    lr, b1, b2, eps, wd = hp
    coef = _f32(0.37) if clip else 1.0
    clip_t = torch.tensor([coef], device="cuda") if clip else None
    for n in (8192, 8193, 8194, 8195, 3):
        for step in ADAM_STEPS:
            w0, m0, v0 = adamw_state(n, step, seed=n + step)
            gen = torch.Generator(device="cuda").manual_seed(n * step)
            g = torch.randn(n, generator=gen, device="cuda").to(gdtype)
            g[::5] = 0
            m, v = m0.clone(), v0.clone()
            if flavour == "fp32":
                w = w0.clone()
                co.adamw_fp32(w, m, v, g, clip_t, lr, b1, b2, eps, wd, step)
            else:
                hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
                lo = torch.empty(n, dtype=torch.int16, device="cuda")
                co.split_fp32(w0, hi, lo)
                check_split(hi, lo, w0)
                if flavour == "split":
                    co.adamw_split(hi, lo, m, v, g, clip_t, lr, b1, b2, eps, wd, step)
                else:
                    hyper = torch.tensor([lr, float(step)], device="cuda")
                    co.adamw_split(hi, lo, m, v, g, clip_t, 10 * lr, b1, b2, eps, wd, step + 7, hyper=hyper)
                w = torch.empty_like(w0)
                co.merge_fp32(hi, lo, w)
                check_split(hi, lo, w)
            check_adamw(w0, m0, v0, g, coef, hp, step, w, m, v)


@pytest.mark.gpu
@pytest.mark.parametrize("hyper", [False, True])
def test_adamw_split_keeps_ties_at_zero_lr(hyper):
    """lr = 0 leaves every weight bit-identical, exact bf16 ties included, and hi still rounds them away from
    zero (the kernel reads lo = -32768 back as a signed remainder)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    n = 4099
    w0, m, v = adamw_state(n, 3, seed=5)
    hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty(n, dtype=torch.int16, device="cuda")
    co.split_fp32(w0, hi, lo)
    assert int((lo == -32768).sum()) > 0
    g = torch.randn(n, device="cuda")
    h = torch.tensor([0.0, 3.0], device="cuda") if hyper else None
    co.adamw_split(hi, lo, m, v, g, None, 1e-3 if hyper else 0.0, 0.9, 0.999, 1e-8, 0.1, 3, hyper=h)
    w = torch.empty_like(w0)
    co.merge_fp32(hi, lo, w)
    assert torch.equal(w.view(torch.int32), w0.view(torch.int32))
    check_split(hi, lo, w)


# ------------------------------------------------------------------------------------------------
# CPU meta-tests: the references agree with autograd, the checkers accept the exact reference and reject mutants
# ------------------------------------------------------------------------------------------------
def _bf(t):
    return t.to(torch.bfloat16)


def test_ln_refs_match_autograd():
    torch.manual_seed(0)
    x, g, b, dy, dres = (t.double() for t in ln_inputs(6, 64, 0, "cpu"))
    for eps in (BLOCK_LN_EPS, FINAL_LN_EPS):
        xr, gr, br = (t.clone().requires_grad_() for t in (x, g, b))
        y = F.layer_norm(xr, (64,), gr, br, eps)
        y.backward(dy)
        y64, mean, rstd, _ = ln_fwd_ref(x, g, b, eps)
        torch.testing.assert_close(y64, y.detach(), rtol=1e-12, atol=1e-12)
        dx, dg, db = ln_bwd_ref(dy, x, g, mean, rstd, dres)
        torch.testing.assert_close(dx, xr.grad + dres, rtol=1e-9, atol=1e-9)
        torch.testing.assert_close(dg, gr.grad, rtol=1e-10, atol=1e-10)
        torch.testing.assert_close(db, br.grad, rtol=1e-12, atol=1e-12)


def test_gelu_refs_match_autograd():
    x = torch.linspace(-9, 9, 2001, dtype=torch.float64, requires_grad=True)
    y = F.gelu(x)
    y.sum().backward()
    # autograd's 1 + erf cancels in float64 too (|error| ~ 1e-16 |x|): hence the absolute term
    torch.testing.assert_close(gelu_ref(x.detach()), y.detach(), rtol=1e-9, atol=1e-14)
    torch.testing.assert_close(dgelu_ref(x.detach()), x.grad, rtol=1e-9, atol=1e-12)


def test_ce_refs_match_autograd():
    logits, target = ce_inputs(8, 37, seed=0, device="cpu")
    for lam, sm in ((1.0, 0.0), (1.0, 0.1), (0.3, 0.1)):
        z = logits.double().requires_grad_()
        loss = lam * F.cross_entropy(z, target, label_smoothing=sm)
        if lam != 1.0:
            loss = loss + (1 - lam) * F.cross_entropy(z, target.flip(0), label_smoothing=sm)
        loss.backward()
        loss64, dl64, _, _, correct = ce_ref(logits, target, lam, sm)
        torch.testing.assert_close(loss64, loss.detach(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(dl64, z.grad, rtol=1e-10, atol=1e-14)
        assert correct == int((logits.double().argmax(1) == target).sum())


def test_adamw_ref_matches_torch_optim():
    torch.manual_seed(0)
    w = torch.randn(100, dtype=torch.float64)
    p = torch.nn.Parameter(w.clone())
    opt = torch.optim.AdamW([p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1)
    m, v = torch.zeros_like(w), torch.zeros_like(w)
    for step in range(1, 5):
        g = torch.randn(100, dtype=torch.float64)
        p.grad = g.clone()
        opt.step()
        w, m, v, _ = adamw_ref(w, m, v, g, 1.0, 1e-3, 0.9, 0.999, 1e-8, 0.1, step)
        torch.testing.assert_close(w, p.detach(), rtol=1e-14, atol=1e-15)


def _ln_case(rows=64, D=64, eps=FINAL_LN_EPS):
    x, g, b, dy, dres = ln_inputs(rows, D, 3, "cpu")
    x = _bf(x.float() * 0.01 + 0.25 * (torch.arange(rows)[:, None] % 2))  # small-variance rows: the eps matters
    return x, g, b, dy, dres, _f32(eps)


def test_ln_fwd_checker_accepts_ref_rejects_mutants():
    x, g, b, _, _, eps = _ln_case()
    y, mean, rstd, _ = ln_fwd_ref(x, g, b, eps)
    check_ln_fwd(x, g, b, eps, _bf(y), mean.float(), rstd.float())
    for name, mutant in (("eps", ln_fwd_ref(x, g, b, eps * 10)), ("D - 1", ln_fwd_ref(x, g, b, eps, ddof=1))):
        y, mean, rstd, _ = mutant
        with pytest.raises(AssertionError):
            check_ln_fwd(x, g, b, eps, _bf(y), mean.float(), rstd.float())


def test_ln_bwd_checker_accepts_ref_rejects_mutants():
    x, g, b, dy, dres, eps = _ln_case(rows=300)
    _, mean, rstd, _ = ln_fwd_ref(x, g, b, eps)
    mean, rstd = mean.float(), rstd.float()
    dx, dg, db = ln_bwd_ref(dy, x, g, mean, rstd, dres)
    dxb = _bf(dx)
    check_ln_bwd(dy, x, g, mean, rstd, dres, dxb, dg.float(), db.float(), dxb.double().sum(0).float())
    with pytest.raises(AssertionError, match="dxsum"):  # summed before rounding to bf16
        check_ln_bwd(dy, x, g, mean, rstd, dres, dxb, dg.float(), db.float(), dx.sum(0).float())
    with pytest.raises(AssertionError, match="dx"):  # a row slot off by one
        check_ln_bwd(dy, x, g, mean, rstd, dres, dxb.roll(1, 0), dg.float(), db.float(), None)


def test_gelu_checkers_accept_ref_reject_mutants():
    grid, _ = finite_bf16_grid()
    check_gelu(grid, _bf(gelu_ref(grid)))
    dg = _bf(torch.randn(grid.shape))
    check_dgelu(grid, dg, _bf(dg.double() * dgelu_ref(grid)))
    tanh_gelu = F.gelu(grid.float(), approximate="tanh")
    with pytest.raises(AssertionError):
        check_gelu(grid, _bf(tanh_gelu))


def test_ce_checker_accepts_ref_rejects_last_tie():
    logits, target = ce_inputs(12, 50, seed=1, device="cpu")
    for lam, sm in ((1.0, 0.0), (0.3, 0.1)):
        loss, dl, _, _, correct = ce_ref(logits, target, lam, sm)
        check_ce(logits, target, lam, sm, loss.float(), _bf(dl), correct)
        last = ce_ref(logits, target, lam, sm, last_tie=True)[4]
        assert last != correct
        with pytest.raises(AssertionError, match="correct"):
            check_ce(logits, target, lam, sm, loss.float(), _bf(dl), last)


def test_adamw_checker_accepts_ref_rejects_float_bias_correction():
    """The checker accepts the float64 step and rejects a bias correction 1 - beta2^t that is 1e-4 off, which is
    what an approximate powf (lg2 / ex2.approx) gives at small t."""
    hp = (_f32(1e-3), _f32(0.9), _f32(0.999), _f32(1e-8), _f32(0.1))
    w0 = torch.randn(1000) * 0.02
    m0, v0 = torch.zeros(1000), torch.zeros(1000)
    g = torch.randn(1000)
    w, m, v, _ = adamw_ref(w0, m0, v0, g, 1.0, *hp, 1)
    check_adamw(w0, m0, v0, g, 1.0, hp, 1, w.float(), m.float(), v.float())
    lr, b1, b2, eps, wd = hp
    bad = w0.double() * (1 - lr * wd) - (lr / (1 - b1)) * m / (v.sqrt() / math.sqrt((1 - b2) * (1 + 1e-4)) + eps)
    with pytest.raises(AssertionError, match="adamw w"):
        check_adamw(w0, m0, v0, g, 1.0, hp, 1, bad.float(), m.float(), v.float())


if __name__ == "__main__":
    _forced_main(sys.argv[1])
