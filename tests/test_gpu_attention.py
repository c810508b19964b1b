"""Attention core (batched wgmma GEMMs + fused softmax) vs the fp32 reference."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _close(got, ref, rel=3e-2):
    """Per-element relative + absolute bound (tests/helpers.py), not a max-normalised one."""
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel)


@pytest.mark.parametrize("B,N,H,hd", [(2, 256, 4, 160), (3, 196, 3, 64), (1, 576, 2, 160)])
def test_attention_fwd_bwd(B, N, H, hd):
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.5).to(torch.bfloat16)
    out, p = co.attention_fwd(qkv, B, N, H, hd)
    outr, pr = to.attention_fwd(qkv.float(), B, N, H, hd)
    _close(p.view(B, H, N, -1)[..., :N], pr)
    _close(out, outr)
    dout = (torch.randn(B * N, D, device="cuda")).to(torch.bfloat16)
    dqkv, cs = co.attention_bwd(dout, qkv, p, B, N, H, hd, want_colsum=True)
    dqkvr, csr = to.attention_bwd(dout.float(), qkv.float(), pr, B, N, H, hd, want_colsum=True)
    _close(dqkv, dqkvr)
    _close(cs, csr, rel=5e-2)


@pytest.mark.parametrize("B,N,H,hd", [(2, 256, 4, 160), (3, 196, 3, 64), (2, 64, 2, 128), (1, 256, 2, 64)])
def test_fused_attention_forward(B, N, H, hd):
    """Fused wgmma kernel (S/P never leave the SM) vs the fp32 reference; with and without the P side output."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    assert co._C.attention_supported(N, hd)
    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.7).to(torch.bfloat16)
    outr, pr = to.attention_fwd(qkv.float(), B, N, H, hd)
    out, p = co.attention_fwd(qkv, B, N, H, hd, need_p=True)
    _close(out, outr)
    _close(p.view(B, H, N, -1)[..., :N], pr)
    out2, p2 = co.attention_fwd(qkv, B, N, H, hd, need_p=False)
    assert p2 is None
    assert torch.equal(out2, out)
    lse = torch.empty(B * H, N, device="cuda")
    out3 = torch.empty_like(out)
    co._C.attention_fwd(qkv, out3, lse, None, B, N, H, hd)
    q, k, _ = qkv.float().view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    lser = torch.logsumexp((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1).reshape(B * H, N)
    assert (lse - lser).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,N,H,hd", [(1, 256, 2, 64), (3, 196, 3, 64), (2, 128, 2, 128), (2, 256, 4, 160)])
def test_fused_attention_backward(B, N, H, hd):
    """attention_sm90.cu (delta kernel + dK/dV role + dQ role) vs the fp32 reference."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    assert co.flash_supported(N, hd)
    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda").to(torch.bfloat16)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd)
    outr, lser = to.attention_fwd_lse(qkv.float(), B, N, H, hd)
    _close(out, outr)
    assert (lse - lser).abs().max().item() < 2e-2
    dqkv, cs = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, want_colsum=True)
    dqkvr, csr = to.attention_bwd_lse(dout.float(), qkv.float(), outr, lser, B, N, H, hd, want_colsum=True)
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        got, ref = dqkv[:, sl].float(), dqkvr[:, sl].float()
        err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        assert err < 3e-2, f"{name}: rel err {err}"
    _close(cs, csr, rel=5e-2)


@pytest.mark.parametrize("B,N,H,hd", [(1, 320, 2, 64), (1, 576, 2, 160), (2, 576, 2, 128)])
def test_fused_attention_long_sequence(B, N, H, hd):
    """Fused forward + backward at N > 256 (336 px config: nine key tiles per query tile) vs the fp32 reference."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda").to(torch.bfloat16)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd)
    outr, lser = to.attention_fwd_lse(qkv.float(), B, N, H, hd)
    _close(out, outr)
    assert (lse - lser).abs().max().item() < 2e-2
    dqkv = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd)
    dqkvr = to.attention_bwd_lse(dout.float(), qkv.float(), outr, lser, B, N, H, hd)
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        got, ref = dqkv[:, sl].float(), dqkvr[:, sl].float()
        err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        assert err < 3e-2, f"{name}: rel err {err}"


@pytest.mark.parametrize("B,N,H,hd", [(2, 256, 4, 160), (3, 196, 3, 64), (5, 160, 2, 128), (40, 256, 8, 160)])
def test_persistent_attention_forward(B, N, H, hd):
    """Forward with the log-sum-exp output through the raw entry point vs the fp32 reference; the last shape has 1280
    work items, several per SM, so CTAs of different items share SMs and follow each other on them."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    assert co._C.attention_supported(N, hd)
    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.7).to(torch.bfloat16)
    out = torch.empty(B * N, D, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B * H, N, device="cuda")
    co._C.attention_fwd(qkv, out, lse, None, B, N, H, hd)
    outr, lser = to.attention_fwd_lse(qkv.float(), B, N, H, hd)
    _close(out, outr)
    assert (lse - lser).abs().max().item() < 2e-2


@pytest.mark.parametrize("B,N,H,hd", [(1, 256, 2, 64), (3, 196, 3, 64), (2, 128, 2, 128), (2, 256, 4, 160),
                                      (40, 256, 8, 160)])
def test_persistent_attention_backward(B, N, H, hd, monkeypatch):
    """Backward with the qkv bias gradient reduced inside the kernels (no separate column-sum launch) vs the fp32
    reference and vs the sums of the stored bf16 gradients; the last shape has many work items per SM."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    D = H * hd
    qkv = (torch.randn(B * N, 3 * D, device="cuda") * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda").to(torch.bfloat16)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd)
    n0 = co.launch_count()
    dqkv, cs = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, want_colsum=True)
    assert co.launch_count() - n0 == 1, "bias-gradient column sums must come out of the backward kernels themselves"
    dqkvr = to.attention_bwd_lse(dout.float(), qkv.float(), out.float(), lse, B, N, H, hd)
    csr = dqkv.float().sum(dim=0)  # sums of the bf16 values that were stored
    assert (cs - csr).abs().max().item() <= 2e-3 * csr.abs().max().item() + 1e-3, "fused qkv bias gradient"
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        got, ref = dqkv[:, sl].float(), dqkvr[:, sl].float()
        err = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-6)
        assert err < 3e-2, f"{name}: rel err {err}"
