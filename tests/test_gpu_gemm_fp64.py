"""The plain wgmma GEMM (csrc/gemm_sm90.cu, gemm_bf16_sm90_kernel) against float64, on poisoned strided operands.

Every one of the 20 non-GLU template instances -- (major_a, major_b) x BLOCK_N x cluster size, plus the four row-scale
instances -- runs at shapes chosen for their edges (M / N / K tails, N % 8 != 0, K below one k-step, an odd m-tile
count, many tiles) and at the three classifier-head GEMMs of a 21841-class model, with every fused epilogue the host
accepts.  A profiler trace asserts which instance ran.

Operands are views into NaN-filled buffers (leading dimension pad8(inner) + 8, eight extra rows, bias[N] NaN for odd
N), so a kernel that reads one element outside the logical matrix returns NaN.  Outputs are views into canvases filled
with a sentinel bit pattern, checked bitwise outside the logical region after every call.  The one store past N that
the kernel makes is the rest of the last 16-byte unit of a row when N % 8 != 0 (the TMA store writes whole 16-byte
units; gemm_sm90.h): those columns [N, pad8(N)) must hold +0 in D.

One error model covers every case (``expected``), in units of u = 2^-24 and of one bf16 ulp of the float64 value:
  accumulator   e_acc = K u (|A| |B|^T)                     (fp32 accumulation of K exact bf16 products)
  v = acc+bias  e_v = e_acc + 2 u |v|
  GELU          max |gelu'| over [v - e_v, v + e_v] * e_v + ERF_TOL (|v| + e_v)
  dGELU         |gelu'(aux)| e_v + ERF_TOL |v| (1 + |aux|) + u |y|
  row scale     |s| e + u |y|
  residual      + u |y|
  bf16 output   + 0.5 bf16_ulp(|y| + e)   (one rounding; the ulp at |y| + e admits a value that crosses 2^k)
  pre-act       the bound of bf16(v)
  column sums   against the float64 sum of the *stored* bf16 outputs, within (rows + 64) u sum |d|
The CPU meta-tests at the end show this checker accepts the exact and an fp32 left-to-right result and rejects
specific wrong kernels at the shapes the GPU tests use.

Also: a NaN tracer (one NaN in A or B must poison exactly its row / column of D), the batched per-head operands of
the un-fused attention path against float64, and schedule / tensor-map-cache invariance.  Every assertion message
carries the worst err / tol ratio, and every GPU test prints its worst ratios (``pytest -rP`` shows them)."""
import functools
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_gpu_memory_bound_fp64 import ERF_TOL, U, KernelTrace, assert_within, bf16_ulp, dgelu_ref, gelu_ref  # noqa: E402
from test_gpu_swiglu import _fp32_sum_bound  # noqa: E402

BF16, F32 = torch.bfloat16, torch.float32
SENTINEL = {BF16: 0x7FA5, F32: 0x7FA5A5A5}  # NaN payloads no kernel writes: any change is a store
INT_OF = {BF16: torch.int16, F32: torch.int32}
NAN = float("nan")

RES_ROW_MOD = 37      # rows of the broadcast residual table (res_row_mod): not a multiple of any tile height
ROWS_PER_SCALE = 49   # rows per row-scale sample: samples straddle the 64-row warpgroup and 128-row tile edges
SCALES = (1.5, 0.0, -0.75, 1.0, 0.3125, 2.0)  # per-sample row scales: zero, one and non-one values

# (M, N, K) and the edge each one targets
SHAPES = [
    (1, 7, 8),            # one row; odd N; K below one 16-wide k-step
    (127, 100, 40),       # one row short of a tile; N % 8 = 4; K below one k-block
    (129, 264, 72),       # odd m-tile count (cluster 2: an empty peer); 8 columns into the last n-tile
    (640, 1000, 200),     # K tail inside a k-block
    (2048, 768, 2056),    # many tiles; num_kb = 33
]
# The classifier head of a 21841-class model at batch 20 and width 320, issued as models/vit.py issues it
# (cuda_ops.linear_fwd / linear_dgrad / linear_wgrad): (major_a, major_b) -> (M, N, K)
CLASSES, HEAD_B, HEAD_D = 21841, 20, 320
HEAD = {(0, 0): (HEAD_B, CLASSES, HEAD_D),   # forward: logits = pooled W^T + b, N = 21841
        (0, 1): (HEAD_B, HEAD_D, CLASSES),   # dgrad: dpooled = dlogits W, K = 21841
        (1, 1): (CLASSES, HEAD_D, HEAD_B)}   # wgrad: dW = dlogits^T pooled, M = 21841

# (major_a, major_b, block_n, cluster, row_scale): the 20 non-GLU instances of gemm_bf16_sm90_kernel
INSTANCES = [(ma, mb, bn, cl, False) for ma in (0, 1) for mb in (0, 1) for bn in (128, 256) for cl in (1, 2)]
INSTANCES += [(0, 0, bn, cl, True) for bn in (128, 256) for cl in (1, 2)]

EPILOGUES = {
    "none": {},
    "bias": dict(bias=True),
    "bias+res": dict(bias=True, residual="full"),
    "bias+res%": dict(bias=True, residual="mod"),
    "bias+gelu+pre": dict(bias=True, act="gelu", pre=True),
    "bias+gelu+pre+res": dict(bias=True, act="gelu", pre=True, residual="full"),
    "dgelu+colsum": dict(act="dgelu", colsum=True),
    "colsum": dict(colsum=True),
}
ROW_SCALE_EPILOGUES = {  # the host takes a row scale only with no activation, aux output or column sums
    "scale": dict(scale=True),
    "bias+scale": dict(bias=True, scale=True),
    "bias+scale+res": dict(bias=True, scale=True, residual="full"),
    "bias+scale+res%": dict(bias=True, scale=True, residual="mod"),
}


def _pad8(n):
    return (n + 7) // 8 * 8


def kernel_name(ma, mb, bn, cl, rs):
    return f"gemm_bf16_sm90_kernel<{ma}, {mb}, {bn}, {4 if bn == 256 else 6}, {cl}, {'true' if rs else 'false'}>"


def _inst_id(inst):
    ma, mb, bn, cl, rs = inst
    return f"{ma}{mb}-bn{bn}-c{cl}" + ("-rowscale" if rs else "")


# ------------------------------------------------------------------------------------------------
# operands, canvases and the error model
# ------------------------------------------------------------------------------------------------
def poisoned(mat):
    """`mat` copied into a NaN-filled buffer with ld = pad8(cols) + 8 and 8 extra rows: (view, ld)."""
    rows, cols = mat.shape
    ld = _pad8(cols) + 8
    buf = torch.full((rows + 8, ld), NAN, dtype=mat.dtype, device=mat.device)
    buf[:rows, :cols] = mat
    return buf[:rows, :cols], ld


def poisoned_vec(vec):
    """A 1-D view into a NaN-filled buffer of pad8(n) + 8 elements: for odd n the kernel's pair read of element n
    finds a NaN, which it must discard."""
    n = vec.numel()
    buf = torch.full((_pad8(n) + 8,), NAN, dtype=vec.dtype, device=vec.device)
    buf[:n] = vec
    return buf[:n]


def sentinel(shape, dtype, device):
    return torch.full(shape, SENTINEL[dtype], dtype=INT_OF[dtype], device=device).view(dtype)


def assert_untouched(name, buf, written):
    """Every element of `buf` outside the boolean mask `written` still holds the sentinel bits."""
    changed = (buf.view(INT_OF[buf.dtype]) != SENTINEL[buf.dtype]) & ~written
    n = int(changed.sum())
    assert n == 0, f"{name}: {n} elements outside the output were written, first at {changed.nonzero()[0].tolist()}"


def mark_output(name, buf, written, r0, c0, rows, cols, tail_zero=True):
    """Marks the output block buf[r0:r0 + rows, c0:c0 + cols] and the rest of the last 16-byte unit of each of its
    rows, columns [cols, pad8(cols)), as written: the TMA store writes whole 16-byte units (gemm_sm90.h).  D must hold
    +0 there (the epilogue zeroes what lies past N); the pre-activation side output holds unspecified values."""
    if tail_zero:
        tail = buf[r0:r0 + rows, c0 + cols:c0 + _pad8(cols)]
        n = int((tail.view(INT_OF[buf.dtype]) != 0).sum())
        assert n == 0, f"{name}: {n} elements of columns [N, pad8(N)) are not +0"
    written[r0:r0 + rows, c0:c0 + _pad8(cols)] = True


class Canvas:
    """A rows x cols output view into a sentinel-filled buffer with ld = pad8(cols) + 8 and 8 extra rows."""

    def __init__(self, rows, cols, dtype, device, zero=False):
        self.rows, self.cols, self.ld = rows, cols, _pad8(cols) + 8
        self.buf = sentinel((rows + 8, self.ld), dtype, device)
        self.view = self.buf[:rows, :cols]
        if zero:
            self.view.zero_()

    def assert_untouched(self, name, tail_zero=True):
        written = torch.zeros(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        if self.buf.dtype == BF16:
            mark_output(name, self.buf, written, 0, 0, self.rows, self.cols, tail_zero)
        else:  # column sums: fp32 atomics, element by element
            written[:self.rows, :self.cols] = True
        assert_untouched(name, self.buf, written)


class Margins:
    """Checks |got - ref| <= tol and keeps the worst err / tol ratio per check, printed at the end of a test."""

    def __init__(self):
        self.worst = {}

    def check(self, name, got, ref, tol):
        err = (got.double() - ref).abs()
        ratio = torch.nan_to_num(err / tol.clamp_min(1e-300), nan=math.inf)
        r = float(ratio.max()) if ratio.numel() else 0.0
        key = name.split(":")[-1].strip()
        self.worst[key] = max(self.worst.get(key, 0.0), r)
        try:
            assert_within(name, got, ref, tol)
        except AssertionError as e:
            raise AssertionError(f"{e}; worst err / tol {r:.3g}") from None

    def colsum(self, name, cs, d, rows):
        """Column sums against the float64 sum of the stored bf16 outputs `d` (summed over dim 0)."""
        d64 = d.double()
        self.check(name, cs, d64.sum(0), (rows + 64) * U * d64.abs().sum(0))

    def report(self):
        print("worst err / tol: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.worst.items())))


class Problem:
    """Logical operands of one (M, N, K) -- A [M, K], B [N, K] and the epilogue inputs, bf16 from a seeded CPU
    generator -- with the float64 product and its accumulator bound."""

    def __init__(self, M, N, K, device):
        self.M, self.N, self.K = M, N, K
        g = torch.Generator().manual_seed(M * 1000003 + N * 1009 + K)

        def bf(*shape, scale=1.0):
            return (torch.randn(*shape, generator=g) * scale).to(BF16).to(device)

        self.A, self.B = bf(M, K), bf(N, K, scale=K ** -0.5)
        self.bias, self.res, self.table, self.aux = bf(N, scale=0.5), bf(M, N), bf(RES_ROW_MOD, N), bf(M, N, scale=1.5)
        n_scales = -(-M // ROWS_PER_SCALE)
        self.scales = torch.tensor([SCALES[i % len(SCALES)] for i in range(n_scales)], dtype=F32, device=device)
        self.acc = self.A.double() @ self.B.double().t()
        self.e_acc = _fp32_sum_bound(self.A, self.B)

    def residual(self, kind):
        if kind == "mod":
            return self.table[torch.arange(self.M, device=self.table.device) % RES_ROW_MOD]
        return self.res

    def row_scales(self):
        return self.scales.double().repeat_interleave(ROWS_PER_SCALE)[:self.M]

    @functools.cached_property
    def poisoned_inputs(self):
        """The epilogue inputs in NaN-filled buffers, built once per problem."""
        return dict(bias=poisoned_vec(self.bias), res=poisoned(self.res), table=poisoned(self.table),
                    aux=poisoned(self.aux), scales=poisoned_vec(self.scales))


def _max_abs_dgelu(lo, hi):
    """max |gelu'(x)| over [lo, hi]: at an end point, or at the extrema of gelu' at x = +-sqrt(2)."""
    m = torch.maximum(dgelu_ref(lo).abs(), dgelu_ref(hi).abs())
    for c in (math.sqrt(2.0), -math.sqrt(2.0)):
        peak = abs(float(dgelu_ref(torch.tensor(c, dtype=torch.float64))))
        m = torch.where((lo <= c) & (c <= hi), m.clamp_min(peak), m)
    return m


def expected(P, bias=False, act="none", residual=None, scale=False, pre=False, colsum=False):
    """float64 reference of one epilogue and the bound on |bf16 output - reference|: (y, tol_y, v, tol_v), v the
    pre-activation acc + bias that the aux output stores.  The error model is in the module docstring."""
    v, e_v = P.acc, P.e_acc
    if bias:
        v = P.acc + P.bias.double()
        e_v = P.e_acc + 2 * U * v.abs()
    tol_v = e_v + 0.5 * bf16_ulp(v.abs() + e_v)
    if act == "gelu":
        y = gelu_ref(v)
        e = _max_abs_dgelu(v - e_v, v + e_v) * e_v + ERF_TOL * (v.abs() + e_v)
    elif act == "dgelu":
        gp = dgelu_ref(P.aux)
        y = v * gp
        e = gp.abs() * e_v + ERF_TOL * v.abs() * (1 + P.aux.double().abs()) + U * y.abs()
    else:
        y, e = v, e_v
    if scale:
        s = P.row_scales()[:, None]
        y = y * s
        e = s.abs() * e + U * y.abs()
    if residual is not None:
        y = y + P.residual(residual).double()
        e = e + U * y.abs()
    return y, e + 0.5 * bf16_ulp(y.abs() + e), v, tol_v


# ------------------------------------------------------------------------------------------------
# one GEMM call on poisoned operands, checked
# ------------------------------------------------------------------------------------------------
def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def operands(P, ma, mb):
    """A and B stored with the given majors (0: K contiguous, 1: M / N contiguous), each in a NaN-filled buffer."""
    return poisoned(P.A if ma == 0 else P.A.t()), poisoned(P.B if mb == 0 else P.B.t())


def run_gemm(P, ops, ma, mb, block_n, cluster, max_ctas=0, bias=False, act="none", residual=None, scale=False,
             pre=False, colsum=False):
    """One gemm_raw call into fresh sentinel canvases: {"d": Canvas, "pre": Canvas | None, "cs": Canvas | None}."""
    co = _co()
    (a, lda), (b, ldb) = ops
    M, N, K = P.M, P.N, P.K
    inp = P.poisoned_inputs
    out = {"d": Canvas(M, N, BF16, a.device), "pre": Canvas(M, N, BF16, a.device) if pre else None,
           "cs": Canvas(1, N, F32, a.device, zero=True) if colsum else None}
    kw = dict(act={"none": co.ACT_NONE, "gelu": co.ACT_GELU, "dgelu": co.ACT_DGELU}[act])
    if bias:
        kw.update(bias=inp["bias"])
    if residual is not None:
        r, ldr = inp["table" if residual == "mod" else "res"]
        kw.update(residual=r, ld_res=ldr, res_row_mod=RES_ROW_MOD if residual == "mod" else 0)
    if act == "dgelu":
        kw.update(aux_in=inp["aux"][0], ld_aux=inp["aux"][1])
    if pre:
        kw.update(aux_out=out["pre"].view, ld_aux_out=out["pre"].ld)
    if colsum:
        kw.update(colsum=out["cs"].view[0])
    if scale:
        kw.update(row_scale=inp["scales"], rows_per_scale=ROWS_PER_SCALE)
    co.gemm_raw(a, lda, ma, b, ldb, mb, out["d"].view, out["d"].ld, M, N, K, block_n=block_n, cluster=cluster,
                max_ctas=max_ctas, **kw)
    return out


def check_outputs(m, case, P, spec, out):
    y, tol, v, tol_v = expected(P, **spec)
    m.check(f"{case}: D", out["d"].view, y, tol)
    out["d"].assert_untouched(f"{case}: D canvas")
    if out["pre"] is not None:
        m.check(f"{case}: pre-activation", out["pre"].view, v, tol_v)
        out["pre"].assert_untouched(f"{case}: pre-activation canvas", tail_zero=False)
    if out["cs"] is not None:
        m.colsum(f"{case}: colsum", out["cs"].view[0], out["d"].view, P.M)
        out["cs"].assert_untouched(f"{case}: colsum[N:]")


def refused(P, spec):
    """The host refuses a residual or aux_in unless N % 8 == 0 (they are read as bf16 pairs of 8-aligned rows)."""
    return P.N % 8 != 0 and (spec.get("residual") is not None or spec.get("act") == "dgelu")


@functools.lru_cache(maxsize=2)
def problem(M, N, K):
    return Problem(M, N, K, "cuda")


# ------------------------------------------------------------------------------------------------
# 1. every instance x shape x epilogue
# ------------------------------------------------------------------------------------------------
CASES = [(inst, shape) for shape in SHAPES for inst in INSTANCES]  # shape-major: one Problem per shape
CASES += [(inst, HEAD[inst[:2]]) for inst in INSTANCES if not inst[4] and inst[:2] in HEAD]


@pytest.mark.gpu
@pytest.mark.parametrize("inst,shape", CASES, ids=[f"{_inst_id(i)}-{'x'.join(map(str, s))}" for i, s in CASES])
def test_instance_against_fp64(inst, shape):
    ma, mb, bn, cl, rs = inst
    P = problem(*shape)
    ops = operands(P, ma, mb)
    m = Margins()
    trace = KernelTrace()
    try:
        for case, spec in (ROW_SCALE_EPILOGUES if rs else EPILOGUES).items():
            if refused(P, spec):
                with pytest.raises(RuntimeError, match="multiple of 8"):
                    run_gemm(P, ops, ma, mb, bn, cl, **spec)
                continue
            out = run_gemm(P, ops, ma, mb, bn, cl, **spec)
            check_outputs(m, case, P, spec, out)
        trace.expect(kernel_name(*inst))
        trace.verify()
    finally:
        trace.stop()
    m.report()


# ------------------------------------------------------------------------------------------------
# 2. NaN tracer: one NaN in A (B) poisons exactly its row (column) of D
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES, ids=_inst_id)
def test_nan_tracer(inst):
    """With act none a NaN at A[r, k] reaches every D[r, n] and nothing else (and B[n, k] every D[m, n]): exact index
    mapping, no tolerance.  Positions at both corners and at the first k of the second k-block."""
    ma, mb, bn, cl, rs = inst
    spec = dict(scale=True) if rs else {}
    for M, N, K in ((129, 264, 72), (640, 1000, 200)):
        P = problem(M, N, K)
        for which, (i, k) in [(w, p) for w in ("A", "B") for p in ((0, 0), (-1, K - 1), ((M if w == "A" else N) // 2,
                                                                                       64))]:
            A, B = P.A.clone(), P.B.clone()
            (A if which == "A" else B)[i, k] = NAN
            ops = (poisoned(A if ma == 0 else A.t()), poisoned(B if mb == 0 else B.t()))
            d = run_gemm(P, ops, ma, mb, bn, cl, **spec)["d"].view
            want = torch.zeros(M, N, dtype=torch.bool, device=d.device)
            if which == "A":
                want[i, :] = True
            else:
                want[:, i] = True
            bad = torch.isnan(d) != want
            assert not bool(bad.any()), (f"{M}x{N}x{K}, NaN at {which}[{i}, {k}]: {int(bad.sum())} elements of D "
                                         f"wrong, first at {bad.nonzero()[0].tolist()}")


# ------------------------------------------------------------------------------------------------
# 3. batched per-head operands of the un-fused attention path
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ntok", [64, 196, 257])
@pytest.mark.parametrize("nb_inner,nb_outer", [(1, 1), (3, 1), (1, 2), (3, 2)])
def test_batched_per_head_operands(nb_inner, nb_outer, ntok):
    """S = Q K^T (K-major / K-major) read in place from a packed qkv buffer, and dV = P^T dO (MN-major / MN-major)
    with per-head column sums (colsum_bi_stride), nb_inner heads x nb_outer images, each problem against float64.
    Batch strides exceed the extents: 8 NaN columns between heads, 8 NaN rows between images."""
    co = _co()
    hd, gap = 64, 8
    hs = hd + gap                                 # head stride (columns)
    rs_ = ntok + gap                              # image stride (rows)
    g = torch.Generator().manual_seed(ntok * 10 + nb_inner * 3 + nb_outer)
    bf = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(BF16).cuda()  # noqa: E731
    m = Margins()
    slabs = [(bo, bi) for bo in range(nb_outer) for bi in range(nb_inner)]

    # S = Q K^T: qkv rows b * rs_ + t; q head h at column h * hs, k head h at nb_inner * hs + h * hs
    q = {s: bf(ntok, hd) for s in slabs}
    k = {s: bf(ntok, hd, scale=hd ** -0.5) for s in slabs}
    ld3 = 2 * nb_inner * hs + gap
    qkv = torch.full((nb_outer * rs_, ld3), NAN, dtype=BF16, device="cuda")
    for (bo, bi) in slabs:
        qkv[bo * rs_:bo * rs_ + ntok, bi * hs:bi * hs + hd] = q[bo, bi]
        qkv[bo * rs_:bo * rs_ + ntok, (nb_inner + bi) * hs:(nb_inner + bi) * hs + hd] = k[bo, bi]
    ldp = _pad8(ntok) + gap
    s_sbi = rs_ * ldp
    for bn in (128, 256):
        for cl in (1, 2):
            s_buf = sentinel((nb_outer * nb_inner * rs_, ldp), BF16, "cuda")
            co.gemm_raw(qkv, ld3, 0, qkv[:, nb_inner * hs:], ld3, 0, s_buf, ldp, ntok, ntok, hd,
                        batch=(nb_inner, nb_outer, hs, rs_ * ld3, hs, rs_ * ld3, s_sbi, nb_inner * s_sbi),
                        block_n=bn, cluster=cl, max_ctas=0)
            written = torch.zeros(s_buf.shape, dtype=torch.bool, device="cuda")
            for (bo, bi) in slabs:
                r0 = (bo * nb_inner + bi) * rs_
                acc = q[bo, bi].double() @ k[bo, bi].double().t()
                tol = _fp32_sum_bound(q[bo, bi], k[bo, bi])
                m.check(f"S bn{bn} c{cl} slab {bo},{bi}: S", s_buf[r0:r0 + ntok, :ntok], acc,
                        tol + 0.5 * bf16_ulp(acc.abs() + tol))
                mark_output(f"S bn{bn} c{cl} slab {bo},{bi}", s_buf, written, r0, 0, ntok, ntok)
            assert_untouched(f"S bn{bn} c{cl}", s_buf, written)

    # dV = P^T dO: P slab (bo, bi) stored [k, m] at rows (bo * nb_inner + bi) * rs_; dO / dV rows b * rs_ + t, head h at
    # column h * hs; column sums of head h at colsum[h * hs + n], summed over the images
    p = {s: bf(ntok, ntok, scale=ntok ** -0.5) for s in slabs}   # stored [K = ntok, M = ntok]
    do = {s: bf(ntok, hd) for s in slabs}                        # stored [K = ntok, N = hd]
    pbuf = torch.full((nb_outer * nb_inner * rs_, ldp), NAN, dtype=BF16, device="cuda")
    ldo = nb_inner * hs + gap
    dobuf = torch.full((nb_outer * rs_, ldo), NAN, dtype=BF16, device="cuda")
    for (bo, bi) in slabs:
        r0 = (bo * nb_inner + bi) * rs_
        pbuf[r0:r0 + ntok, :ntok] = p[bo, bi]
        dobuf[bo * rs_:bo * rs_ + ntok, bi * hs:bi * hs + hd] = do[bo, bi]
    for bn in (128, 256):
        for cl in (1, 2):
            out = sentinel((nb_outer * rs_, ldo), BF16, "cuda")
            cs = sentinel((ldo,), F32, "cuda")
            for bi in range(nb_inner):
                cs[bi * hs:bi * hs + hd] = 0
            co.gemm_raw(pbuf, ldp, 1, dobuf, ldo, 1, out, ldo, ntok, hd, ntok,
                        batch=(nb_inner, nb_outer, s_sbi, nb_inner * s_sbi, hs, rs_ * ldo, hs, rs_ * ldo),
                        colsum=cs, colsum_bi_stride=hs, block_n=bn, cluster=cl, max_ctas=0)
            written = torch.zeros(out.shape, dtype=torch.bool, device="cuda")
            cs_written = torch.zeros(cs.shape, dtype=torch.bool, device="cuda")
            for (bo, bi) in slabs:
                a, b = p[bo, bi].t(), do[bo, bi].t()      # logical A [M, K], B [N, K]
                acc = a.double() @ b.double().t()
                tol = _fp32_sum_bound(a, b)
                got = out[bo * rs_:bo * rs_ + ntok, bi * hs:bi * hs + hd]
                m.check(f"dV bn{bn} c{cl} slab {bo},{bi}: dV", got, acc, tol + 0.5 * bf16_ulp(acc.abs() + tol))
                mark_output(f"dV bn{bn} c{cl} slab {bo},{bi}", out, written, bo * rs_, bi * hs, ntok, hd)
            for bi in range(nb_inner):
                stored = torch.cat([out[bo * rs_:bo * rs_ + ntok, bi * hs:bi * hs + hd] for bo in range(nb_outer)])
                m.colsum(f"dV bn{bn} c{cl} head {bi}: colsum", cs[bi * hs:bi * hs + hd], stored, nb_outer * ntok)
                cs_written[bi * hs:bi * hs + hd] = True
            assert_untouched(f"dV bn{bn} c{cl}", out, written)
            assert_untouched(f"dV colsum bn{bn} c{cl}", cs, cs_written)
    m.report()


# ------------------------------------------------------------------------------------------------
# 4. schedule and tensor-map cache invariance
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ma,mb", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_schedule_invariance(ma, mb):
    """1000 x 1000 x 200 at BLOCK_N 128: 64 tiles, num_kb = 4 against a 6-stage ring, so with a few persistent CTAs
    the ring's phase and the staging-buffer flip carry across tiles.  D and the pre-activation must be bitwise the
    all-SM result (max_ctas = 0, cluster 1), the column sums equal up to atomic order (checked against float64)."""
    P = problem(1000, 1000, 200)
    ops = operands(P, ma, mb)
    m = Margins()
    for case in ("bias+gelu+pre+res", "dgelu+colsum"):
        spec = EPILOGUES[case]
        base = run_gemm(P, ops, ma, mb, 128, 1, **spec)
        check_outputs(m, f"{case} all SMs", P, spec, base)
        for cl in (1, 2):
            for max_ctas in (0, 1, 3, 8):
                name = f"{case} cluster {cl} max_ctas {max_ctas}"
                out = run_gemm(P, ops, ma, mb, 128, cl, max_ctas=max_ctas, **spec)
                for key in ("d", "pre"):
                    if out[key] is not None:
                        assert torch.equal(out[key].buf.view(torch.int16), base[key].buf.view(torch.int16)), \
                            f"{name}: {key} differs from the all-SM result"
                if out["cs"] is not None:
                    m.colsum(f"{name}: colsum", out["cs"].view[0], out["d"].view, P.M)
                    out["cs"].assert_untouched(f"{name}: colsum[N:]")
    m.report()


@pytest.mark.gpu
def test_tensor_map_cache_tells_layouts_apart():
    """The tensor maps are cached by (base pointer, extents, strides, box): two calls on the same base pointers with
    another ld, then with a shorter K (the columns past it NaN), then with a narrower N, each against float64."""
    co = _co()
    m = Margins()
    M, N, K = 300, 200, 136
    big = Problem(M, N, K, "cuda")
    abuf = torch.empty(M * (K + 64) + 64, dtype=BF16, device="cuda")
    bbuf = torch.empty(N * (K + 64) + 64, dtype=BF16, device="cuda")
    dbuf = sentinel((M + 8, N + 8), BF16, "cuda")
    for lda, k, n in ((K + 8, K, N), (K + 64, K, N), (K + 64, 72, N), (K + 64, 72, 104)):
        P = Problem(M, n, k, "cuda") if (k, n) != (K, N) else big
        abuf.fill_(NAN)
        bbuf.fill_(NAN)
        a = abuf[:M * lda].view(M, lda)
        b = bbuf[:n * lda].view(n, lda)
        a[:, :k], b[:, :k] = P.A, P.B
        dbuf.view(torch.int16).fill_(SENTINEL[BF16])
        co.gemm_raw(a, lda, 0, b, lda, 0, dbuf, N + 8, M, n, k, block_n=128, cluster=1, max_ctas=0)
        y, tol, _, _ = expected(P)
        m.check(f"ld {lda} K {k} N {n}: D", dbuf[:M, :n], y, tol)
        written = torch.zeros(dbuf.shape, dtype=torch.bool, device="cuda")
        mark_output(f"ld {lda} K {k} N {n}: D", dbuf, written, 0, 0, M, n)
        assert_untouched(f"ld {lda} K {k} N {n}: D canvas", dbuf, written)
    m.report()


# ------------------------------------------------------------------------------------------------
# 5. CPU meta-tests: the checker accepts correct results and rejects specific wrong kernels
# ------------------------------------------------------------------------------------------------
META_SHAPES = [(127, 100, 40), (640, 1000, 200)]


def _bf(t):
    return t.to(BF16)


def _fp32_left_to_right(P):
    """A left-to-right fp32 accumulation; each bf16 product is exact in fp32."""
    A, B = P.A.float(), P.B.float()
    acc = torch.zeros(P.M, P.N)
    for k in range(P.K):
        acc += A[:, k:k + 1] * B[:, k]
    return acc


def _fp32_epilogue(P, acc, bias=False, act="none", residual=None, scale=False, pre=False, colsum=False):
    """The kernel's epilogue arithmetic in fp32 on the fp32 accumulator `acc`: (y, v), each to be rounded to bf16
    once."""
    v = acc + P.bias.float() if bias else acc
    if act == "gelu":
        y = torch.nn.functional.gelu(v)
    elif act == "dgelu":
        x = P.aux.float()
        y = v * (0.5 * torch.erfc(-x / math.sqrt(2.0)) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi))
    else:
        y = v
    if scale:
        y = y * P.row_scales().float()[:, None]
    if residual is not None:
        y = y + P.residual(residual).float()
    return y, v


@pytest.mark.parametrize("M,N,K", META_SHAPES)
def test_checker_accepts_fp64_and_fp32_results(M, N, K):
    P = Problem(M, N, K, "cpu")
    acc = _fp32_left_to_right(P)
    m = Margins()
    for case, spec in {**EPILOGUES, **ROW_SCALE_EPILOGUES}.items():
        y, tol, v, tol_v = expected(P, **spec)
        y32, v32 = _fp32_epilogue(P, acc, **spec)
        for name, got_y, got_v in (("fp64", y, v), ("fp32", y32, v32)):
            d = _bf(got_y)
            m.check(f"{case} {name}: D", d, y, tol)
            if spec.get("pre"):
                m.check(f"{case} {name}: pre-activation", _bf(got_v), v, tol_v)
            if spec.get("colsum"):
                m.colsum(f"{case} {name}: colsum", d.double().sum(0).float(), d, M)
    m.report()


@pytest.mark.parametrize("M,N,K", META_SHAPES)
def test_checker_rejects_mutants(M, N, K):
    P = Problem(M, N, K, "cpu")
    m = Margins()
    E = {**EPILOGUES, **ROW_SCALE_EPILOGUES}

    def rejects(case, got):
        y, tol, _, _ = expected(P, **E[case])
        with pytest.raises(AssertionError, match="worst err / tol"):
            m.check(case, got, y, tol)

    k0 = (K - 1) // 16 * 16  # the last 16-wide k-step
    rejects("none", _bf(P.A.double()[:, :k0] @ P.B.double()[:, :k0].t()))
    rejects("bias", _bf(P.acc + torch.cat([P.bias[1:], P.bias[:1]]).double()))
    v = P.acc + P.bias.double()
    rejects("bias+gelu+pre", _bf(gelu_ref(_bf(v))))
    rejects("bias+res", _bf(_bf(v).double() + P.res.double()))
    rejects("bias+scale+res", _bf((v + P.res.double()) * P.row_scales()[:, None]))
    d = _bf(expected(P, **E["colsum"])[0])
    skip = torch.arange(M) % 32 != 31
    with pytest.raises(AssertionError, match="worst err / tol"):
        m.colsum("colsum", d[skip].double().sum(0).float(), d, M)
