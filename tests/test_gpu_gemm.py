"""wgmma GEMM vs an fp32 PyTorch reference (all operand majors, tile widths, fused epilogues)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _ops():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(torch.bfloat16)


def _close(got, ref, rel=2e-2):
    """Per-element relative + absolute bound (tests/helpers.py), not a max-normalised one."""
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 768, 320), (1000, 520, 200), (128, 1000, 5120),
                                   (2048, 5120, 5120)])
@pytest.mark.parametrize("block_n", [128, 256])
def test_nt(M, N, K, block_n):
    ops = _ops()
    x, w = _rand(M, K), _rand(N, K, scale=0.05)
    y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm_raw(x, K, 0, w, K, 0, y, N, M, N, K, block_n=block_n)
    _close(y, x.float() @ w.float().t())


@pytest.mark.parametrize("M,N,K", [(512, 768, 320), (1000, 520, 200), (2048, 5120, 1024)])
def test_dgrad_nn(M, N, K):
    ops = _ops()
    dy, w = _rand(M, N), _rand(N, K, scale=0.05)
    dx = ops.linear_dgrad(dy, w)
    _close(dx, dy.float() @ w.float())


@pytest.mark.parametrize("T,N,K", [(512, 768, 320), (1000, 520, 200), (4096, 1024, 512)])
def test_wgrad_tn(T, N, K):
    ops = _ops()
    dy, x = _rand(T, N), _rand(T, K)
    dw = ops.linear_wgrad(dy, x)
    _close(dw, dy.float().t() @ x.float())


def test_mn_major_a_k_major_b():
    ops = _ops()
    M, N, K = 384, 512, 256
    at, b = _rand(K, M), _rand(N, K)  # A stored transposed: [K, M]
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm_raw(at, M, 1, b, K, 0, d, N, M, N, K)
    _close(d, at.float().t() @ b.float().t())


@pytest.mark.parametrize("K", [512, 2048])  # 512: stand-alone GELU kernels, 2048: fused in the GEMM epilogue
def test_fused_epilogues(K):
    ops = _ops()
    from vit_10b_fsdp_example_b200.ops import torch_ops

    M, N = 640, 1024
    x, w, b, r = _rand(M, K), _rand(N, K, scale=0.05), _rand(N), _rand(M, N)
    y, pre = ops.linear_fwd(x, w, b, act="gelu", residual=r, want_preact=True)
    yr, prer = torch_ops.linear_fwd(x.float(), w.float(), b.float(), act="gelu", residual=r.float(), want_preact=True)
    _close(pre, prer)
    _close(y, yr)
    # broadcast residual (pos_embed style)
    tab = _rand(128, N)
    y2 = ops.linear_fwd(x, w, b, residual=tab, res_row_mod=128)
    y2r = torch_ops.linear_fwd(x.float(), w.float(), b.float(), residual=tab.float(), res_row_mod=128)
    _close(y2, y2r)
    # dgelu + column sums
    N2 = K  # reduction length of the dgrad GEMM decides fused vs stand-alone dGELU
    dy, w2, u = _rand(M, N2), _rand(N2, 768, scale=0.05), _rand(M, 768)
    dx, cs = ops.linear_dgrad(dy, w2, dgelu_preact=u, want_colsum=True)
    dxr, csr = torch_ops.linear_dgrad(dy.float(), w2.float(), dgelu_preact=u.float(), want_colsum=True)
    _close(dx, dxr)
    _close(cs, csr, rel=3e-2)


def test_persistent_many_tiles_and_repeat():
    ops = _ops()
    M, N, K = 8192, 4096, 1024
    x, w = _rand(M, K), _rand(N, K, scale=0.05)
    ref = x.float() @ w.float().t()
    for _ in range(3):
        y = ops.linear_fwd(x, w)
        _close(y, ref)


@pytest.mark.parametrize("which", ["qkv_fwd", "fc2_fwd", "fc2_dgrad_dgelu", "fc1_wgrad"])
def test_real_vit10b_shapes(which):
    """The GEMMs of one ViT-10B block at the benchmarked size (32768 tokens, D 5120, FFN 20480) against an fp32
    reference computed on a strided sample of output rows / columns (the full fp32 product would take minutes)."""
    ops = _ops()
    T, D, F = 32768, 5120, 20480
    rows = torch.arange(0, T, 257, device="cuda")
    if which == "qkv_fwd":
        x, w, b = _rand(T, D), _rand(3 * D, D, scale=0.02), _rand(3 * D)
        y = ops.linear_fwd(x, w, b)
        _close(y[rows], x[rows].float() @ w.float().t() + b.float())
    elif which == "fc2_fwd":  # K = 20480, residual epilogue
        g, w, b, r = _rand(T, F, scale=0.5), _rand(D, F, scale=0.01), _rand(D), _rand(T, D)
        y = ops.linear_fwd(g, w, b, residual=r)
        _close(y[rows], g[rows].float() @ w.float().t() + b.float() + r[rows].float())
    elif which == "fc2_dgrad_dgelu":  # MN-major B, dGELU epilogue + column sums
        from vit_10b_fsdp_example_b200.ops import torch_ops as to

        dy, w, u = _rand(T, D), _rand(D, F, scale=0.02), _rand(T, F)
        du, cs = ops.linear_dgrad(dy, w, dgelu_preact=u, want_colsum=True)
        ref = (dy[rows].float() @ w.float()) * to.dgelu(u[rows].float())
        _close(du[rows], ref)
        _close(cs, du.float().sum(dim=0), rel=2e-2)
    else:  # wgrad: both operands MN-major, reduction over all 32768 tokens
        du, h = _rand(T, F, scale=0.5), _rand(T, D)
        dw = ops.linear_wgrad(du, h)
        cols = torch.arange(0, F, 113, device="cuda")
        _close(dw[cols], du[:, cols].float().t() @ h.float())
