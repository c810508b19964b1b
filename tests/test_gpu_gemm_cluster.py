"""2-CTA clusters with a multicast B tile vs one CTA per tile: same MMAs in the same order per tile, so every output is
bitwise identical; only the fp32 atomic column sums may differ in the last bits (different arrival order).
Covers all operand majors and tile widths, odd and single m-tile counts (the surplus CTA of the last pair), batched
operands, every fused epilogue and the ViT-10B block GEMMs at the benchmarked size."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu


def _ops():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(torch.bfloat16)


def _both(fn):
    """fn() under cluster 1 and cluster 2; results cloned so buffers written in place are compared too."""
    ops = _ops()
    out = []
    try:
        for c in (1, 2):
            ops.set_gemm_cluster(c)
            r = fn()
            out.append(tuple(t.clone() for t in r) if isinstance(r, tuple) else (r.clone(),))
    finally:
        ops.set_gemm_cluster(0)
    return out


def _same(r1, r2, colsum_idx=()):
    for i, (a, b) in enumerate(zip(r1, r2)):
        if i in colsum_idx:
            tol = 1e-5 * max(1.0, a.abs().max().item())
            assert torch.allclose(a, b, rtol=1e-5, atol=tol), (i, (a - b).abs().max().item())
        else:
            assert torch.equal(a, b), (i, (a.float() - b.float()).abs().max().item())


@pytest.mark.parametrize("major_a,major_b", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M,N,K", [(128, 384, 320), (640, 520, 200), (1000, 256, 512), (520, 1000, 128)])
def test_majors_and_odd_m_tiles(major_a, major_b, block_n, M, N, K):
    """M = 128: one m-tile (the pair's second CTA is wholly below the matrix); 640 / 520: five m-tiles."""
    ops = _ops()
    a = _rand(M, K) if major_a == 0 else _rand(K, M)
    b = _rand(N, K, scale=0.05) if major_b == 0 else _rand(K, N, scale=0.05)
    ldd = (N + 7) // 8 * 8

    def run():
        d = torch.full((M, ldd), 7.0, device="cuda", dtype=torch.bfloat16)
        ops.gemm_raw(a, a.shape[1], major_a, b, b.shape[1], major_b, d, ldd, M, N, K, block_n=block_n)
        return d

    r1, r2 = _both(run)
    _same(r1, r2)
    ref = (a.float() if major_a == 0 else a.float().t()) @ (b.float().t() if major_b == 0 else b.float())
    assert (r1[0][:, :N].float() - ref).abs().max().item() <= 0.03 * ref.abs().max().item() + 0.05


@pytest.mark.parametrize("ntok", [128, 196, 320])  # 1, 2 and 3 m-tiles per (image, head) problem
def test_batched_attention_operands(ntok):
    """Per-(image, head) batched problems addressed in place inside a packed qkv buffer, as the un-fused attention
    path runs them: S = Q K^T (K-major / K-major) and dV = P^T dO (MN-major / MN-major) with per-head column sums."""
    ops = _ops()
    B, H, hd = 3, 2, 64
    D = H * hd
    ldp = (ntok + 7) // 8 * 8
    qkv = _rand(B * ntok, 3 * D)
    ld3 = qkv.stride(0)
    p = _rand(B * H, ntok, ldp, scale=0.1)
    dout = _rand(B * ntok, D)

    def scores():
        s = torch.zeros(B * H, ntok, ldp, device="cuda", dtype=torch.bfloat16)
        ops.gemm_raw(qkv[:, :D], ld3, 0, qkv[:, D:2 * D], ld3, 0, s, ldp, ntok, ntok, hd,
                     batch=(H, B, hd, ntok * ld3, hd, ntok * ld3, ntok * ldp, H * ntok * ldp))
        return s

    def dv():
        out = torch.empty(B * ntok, D, device="cuda", dtype=torch.bfloat16)
        cs = torch.zeros(D, device="cuda", dtype=torch.float32)
        ops.gemm_raw(p, ldp, 1, dout, D, 1, out, D, ntok, hd, ntok,
                     batch=(H, B, ntok * ldp, H * ntok * ldp, hd, ntok * D, hd, ntok * D), colsum=cs,
                     colsum_bi_stride=hd)
        return out, cs

    r1, r2 = _both(scores)
    _same(r1, r2)
    r1, r2 = _both(dv)
    _same(r1, r2, colsum_idx=(1,))


@pytest.mark.parametrize("K", [512, 2048])  # 512: stand-alone GELU kernels, 2048: fused in the GEMM epilogue
def test_fused_epilogues(K):
    ops = _ops()
    M, N = 640, 1024
    x, w, b, r = _rand(M, K), _rand(N, K, scale=0.05), _rand(N), _rand(M, N)
    tab = _rand(128, N)
    dy, w2, u = _rand(M, K), _rand(K, 768, scale=0.05), _rand(M, 768)
    cases = [
        (lambda: ops.linear_fwd(x, w, b), ()),
        (lambda: ops.linear_fwd(x, w, b, residual=r), ()),
        (lambda: ops.linear_fwd(x, w, b, act="gelu", residual=r, want_preact=True), ()),
        (lambda: ops.linear_fwd(x, w, b, residual=tab, res_row_mod=128), ()),
        (lambda: ops.linear_dgrad(dy, w2, dgelu_preact=u, want_colsum=True), (1,)),
        (lambda: ops.linear_dgrad(dy, w2), ()),
        (lambda: ops.linear_wgrad(dy, x), ()),
    ]
    for fn, cs in cases:
        r1, r2 = _both(fn)
        _same(r1, r2, colsum_idx=cs)


def test_vit10b_block_gemms():
    """The 12 GEMMs of one ViT-10B block at 32768 tokens, called the way models/vit.py calls them."""
    import bench_gemm

    gemms = bench_gemm.block_gemms(_ops(), 32768, 5120, 20480)
    for name, (_, ours, _) in gemms.items():
        r1, r2 = _both(ours)
        _same(r1, r2, colsum_idx=(1,) if name == "fc2_dgrad" else ())
        del r1, r2
    del gemms
    torch.cuda.empty_cache()
