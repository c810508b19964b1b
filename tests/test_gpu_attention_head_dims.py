"""Fused attention at the head dims beyond 64 / 128 / 160: tile widths 32, 48, 80, 96, 112 and 144, with the head dims
40, 72, 88, 104 and 136 zero-padded to the next multiple of 16 (csrc/attention_sm90.cuh, TileCfg).

The kernel entry points (_C.attention_fwd / attention_bwd, cuda_ops.attention_fwd_lse / attention_bwd_lse) take all of
them.  The model routes a head dim through the fused pair only where _C.attention_supported says so (ROUTED below, the
measured policy in csrc/attention_sm90.cu); the model-level test forces the route to cover the others."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

NEW_WIDTHS = [32, 48, 80, 96, 112, 144]
PADDED = [40, 72, 88, 104, 136]
NEW_HEAD_DIMS = sorted(NEW_WIDTHS + PADDED)
KERNEL_HEAD_DIMS = {32, 40, 48, 64, 72, 80, 88, 96, 104, 112, 128, 136, 144, 160}
ROUTED = {32, 40, 48, 64, 128, 160}
KEY = 0x0DD_BA11


def _close(got, ref, rel=3e-2, what=""):
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel, what=what)


def _close_max(got, ref, what, rel=3e-2):
    err = (got.float() - ref.float()).abs().max().item() / (ref.float().abs().max().item() + 1e-6)
    assert err < rel, f"{what}: rel err {err}"


def _parts(D):
    return (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D)))


@pytest.mark.parametrize("N", [256, 196, 576])
@pytest.mark.parametrize("hd", NEW_HEAD_DIMS)
def test_forward_and_backward_match_the_fp32_reference(hd, N):
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    B, H = (1, 2) if N == 576 else (2, 3)
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(hd * 1000 + N)
    qkv = (torch.randn(B * N, 3 * D, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    outr, lser = to.attention_fwd_lse(qkv.float(), B, N, H, hd)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd)
    _close(out, outr, what="out")
    assert (lse - lser).abs().max().item() < 2e-2
    # the forward with the probability side output
    ldp = (N + 7) // 8 * 8
    p = torch.zeros(B * H, N, ldp, device="cuda", dtype=torch.bfloat16)
    out_p = torch.empty_like(out)
    co._C.attention_fwd(qkv, out_p, None, p, B, N, H, hd)
    _, pr = to.attention_fwd(qkv.float(), B, N, H, hd)
    _close(p[..., :N].reshape(B, H, N, N), pr, what="P")
    assert torch.equal(out_p, out)
    n0 = co.launch_count()
    dqkv, cs = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, want_colsum=True)
    assert co.launch_count() - n0 == 1, "bias-gradient column sums must come out of the backward kernels themselves"
    dqkvr = to.attention_bwd_lse(dout.float(), qkv.float(), outr, lser, B, N, H, hd)
    for name, sl in _parts(D):
        _close_max(dqkv[:, sl], dqkvr[:, sl], name)
    csr = dqkv.float().sum(dim=0)  # sums of the bf16 values that were stored
    assert (cs - csr).abs().max().item() <= 2e-3 * csr.abs().max().item() + 1e-3, "fused qkv bias gradient"


def _heads_mask(B, N, H, hd, parts, h, extra):
    """Boolean [B*N, parts*H*hd + extra] mask of the columns of head h in each of the parts."""
    m = torch.zeros(B * N, parts * H * hd + extra, dtype=torch.bool, device="cuda")
    for i in range(parts):
        m[:, (i * H + h) * hd:(i * H + h + 1) * hd] = True
    return m


def _run_raw(co, qkv, dout, B, N, H, hd):
    """Forward + backward through the raw entry points into NaN-filled outputs.  Each output sits at the start of a
    larger NaN buffer, so a store past its last column is caught too."""
    D = H * hd
    pad = 64
    out_buf = torch.full((B * N * D + pad,), float("nan"), device="cuda", dtype=torch.bfloat16)
    lse = torch.full((B * H, N), float("nan"), device="cuda")
    out = out_buf[:B * N * D].view(B * N, D)
    co._C.attention_fwd(qkv, out, lse, None, B, N, H, hd, 0.0, 0)
    d_buf = torch.full((B * N * 3 * D + pad,), float("nan"), device="cuda", dtype=torch.bfloat16)
    dqkv = d_buf[:B * N * 3 * D].view(B * N, 3 * D)
    delta = torch.full((B * H, N), float("nan"), device="cuda")
    cs = torch.zeros(3 * D, device="cuda")
    co._C.attention_bwd(qkv, dout, out, lse, delta, dqkv, cs, B, N, H, hd, 0.0, 0)
    torch.cuda.synchronize()
    assert torch.isnan(out_buf[B * N * D:]).all() and torch.isnan(d_buf[B * N * 3 * D:]).all(), "store past the end"
    for name, t in (("out", out), ("lse", lse), ("dqkv", dqkv)):
        assert not torch.isnan(t).any(), f"{name} not fully written"
    return out, lse, dqkv


@pytest.mark.parametrize("hd", PADDED)
def test_padded_kernels_stay_inside_their_head(hd):
    """A zero-padded head must read and write its hd columns only.  The qkv rows carry 8 spare columns past the last head
    of v.  For every head h, everything outside head h (the neighbouring heads, the spare columns, the next token's q)
    is replaced by large values: head h's out, lse, dq, dk and dv must stay bitwise the same.  Outputs start as NaN and
    must be fully overwritten, with nothing stored past their end."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    B, N, H = 2, 196, 3
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(hd)
    base = (torch.randn(B * N, 3 * D + 8, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dbase = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    out, lse, dqkv = _run_raw(co, base[:, :3 * D], dbase, B, N, H, hd)
    outr, lser = to.attention_fwd_lse(base[:, :3 * D].float(), B, N, H, hd)
    _close(out, outr, what="out")
    dqkvr = to.attention_bwd_lse(dbase.float(), base[:, :3 * D].float(), outr, lser, B, N, H, hd)
    for name, sl in _parts(D):
        _close_max(dqkv[:, sl], dqkvr[:, sl], name)
    for h in range(H):
        keep = _heads_mask(B, N, H, hd, 3, h, 8)
        dkeep = _heads_mask(B, N, H, hd, 1, h, 0)
        big = (torch.randn(base.shape, device="cuda", generator=g) * 64).to(torch.bfloat16)
        qkv_h = torch.where(keep, base, big)
        dout_h = torch.where(dkeep, dbase, (torch.randn(dbase.shape, device="cuda", generator=g) * 64).to(torch.bfloat16))
        out_h, lse_h, dqkv_h = _run_raw(co, qkv_h[:, :3 * D], dout_h, B, N, H, hd)
        cols = slice(h * hd, (h + 1) * hd)
        assert torch.equal(out_h[:, cols], out[:, cols]), f"head {h}: out"
        assert torch.equal(lse_h.view(B, H, N)[:, h], lse.view(B, H, N)[:, h]), f"head {h}: lse"
        for i, name in enumerate(("dq", "dk", "dv")):
            c = slice(i * D + h * hd, i * D + (h + 1) * hd)
            assert torch.equal(dqkv_h[:, c], dqkv[:, c]), f"head {h}: {name}"


# ---- attention dropout at the new widths ----
def _ref_mask(co, B, N, H, p, key):
    ldp = (N + 7) // 8 * 8
    ones = torch.ones(B * H, N, ldp, device="cuda", dtype=torch.bfloat16)
    return (co.dropout(ones, p, key) != 0)[..., :N].reshape(B, H, N, N)


@pytest.mark.parametrize("hd", NEW_HEAD_DIMS)
def test_fused_dropout_matches_the_unfused_route(hd):
    """The fused pair with drop=(p, key) against the un-fused route (materialised P + Philox dropout kernel) on the
    same mask."""
    from helpers import assert_close_elementwise
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    B, N, H, p = 2, 196, 3, 0.1
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(hd)
    qkv = (torch.randn(B * N, 3 * D, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    drop = (p, KEY)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd, drop=drop)
    n0 = co.launch_count()
    dqkv, cs = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, want_colsum=True, drop=drop)
    assert co.launch_count() - n0 == 1
    outu, P = co.attention_fwd(qkv, B, N, H, hd, drop=drop)
    dqkvu, csu = co.attention_bwd(dout, qkv, P, B, N, H, hd, want_colsum=True, drop=drop)
    assert_close_elementwise(out, outu, rtol=3e-2, atol_rel=3e-2, what="out vs un-fused")
    for name, sl in _parts(D):
        _close_max(dqkv[:, sl], dqkvu[:, sl], name + " vs un-fused")
    assert_close_elementwise(cs, csu, rtol=5e-2, atol_rel=5e-2, what="qkv bias grad vs un-fused")
    # the forward without the log-sum-exp gives the same output
    out2 = torch.empty_like(out)
    co._C.attention_fwd(qkv, out2, None, None, B, N, H, hd, p, KEY)
    assert torch.equal(out2, out)


@pytest.mark.parametrize("B,N,H,hd", [(1, 70, 2, 72), (2, 130, 1, 136), (1, 40, 3, 40)])
def test_dropout_mask_read_out_at_padded_head_dims(B, N, H, hd):
    """Q = K = 0 makes P uniform; one-hot V rows read the mask out through O (O[q, j] = s / N * M[q, j]) and one-hot dO
    rows through dV (dV[k, j] = s / N * M[j, k])."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    p = 0.3
    scale = 1.0 / (1.0 - int(p * 65536.0 + 0.5) / 65536.0)
    zeros = torch.zeros(B, H, N, hd, device="cuda")
    eye = torch.zeros(B, H, N, hd, device="cuda")
    eye[..., torch.arange(N), torch.arange(N)] = 1.0
    qkv = torch.stack([zeros, zeros, eye], 0).permute(1, 3, 0, 2, 4).reshape(B * N, 3 * H * hd)
    qkv = qkv.to(torch.bfloat16).contiguous()
    dout = eye.permute(0, 2, 1, 3).reshape(B * N, H * hd).to(torch.bfloat16)
    m = _ref_mask(co, B, N, H, p, KEY)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd, drop=(p, KEY))
    dqkv = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, drop=(p, KEY))
    o = out.float().view(B, N, H, hd).permute(0, 2, 1, 3)
    assert torch.equal(o[..., :N] != 0, m)
    assert not o[..., N:].any()
    kept = o[..., :N][m]
    assert torch.allclose(kept, torch.full_like(kept, scale / N), rtol=1e-2)
    dv = dqkv.float().view(B, N, 3, H, hd)[:, :, 2].permute(0, 2, 1, 3)
    assert torch.equal(dv[..., :N] != 0, m.transpose(-1, -2))


# ---- model level ----
def _full_grads(model):
    return {u.name: u.shard_grad.float().clone() for u in model.all_units}


@pytest.mark.parametrize("dim,att_dropout", [(160, 0.0), (176, 0.0), (176, 0.1)])
def test_flash_attention_engine_path_at_padded_head_dims(dim, att_dropout, monkeypatch):
    """Same model, same data: loss and gradients with the fused attention pair match the un-fused route to bf16 noise,
    for hd = 80 (embed 160) and hd = 88 (embed 176, zero-padded to 96), with and without kept blocks, and once with
    attention dropout (same Philox masks on both routes).  The fused arm routes these head dims through the fused pair
    (the default routing does not); the un-fused arm also turns the fused forward kernel off, so the two arms share no
    attention kernel."""
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = ViTConfig(image_size=224, patch_size=14, embed_dim=dim, num_heads=2, num_blocks=2, mlp_ratio=4.0,
                    num_classes=96, att_dropout=att_dropout)
    dev = torch.device("cuda")
    routed = co._C.attention_supported
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 3, 224, 224, generator=g).to(dev)
    y = torch.randint(0, 96, (4,), generator=g).to(dev)
    res = []
    for flash in (False, True):
        monkeypatch.setattr(co, "FLASH_ATTENTION", flash)
        monkeypatch.setattr(co, "FUSED_ATTENTION", flash)
        monkeypatch.setattr(co._C, "attention_supported",
                            (lambda n, hd: n % 2 == 0 and hd in KERNEL_HEAD_DIMS) if flash else routed)
        assert co.use_flash(cfg.num_patches, cfg.head_dim) == flash
        for keep in (0, 2):
            model = FSDPViT(cfg, device=dev, dtype=torch.bfloat16, seed=4, ckpt_keep_blocks=keep)
            loss = model.forward_backward(x, y).item()
            res.append((loss, _full_grads(model)))
    for loss, grads in res[1:]:
        assert abs(loss - res[0][0]) < 2e-3
        for k in grads:
            a, b = res[0][1][k], grads[k]
            assert (a - b).norm().item() <= 3e-2 * a.norm().item() + 1e-6, k


def test_routing_takes_exactly_the_routed_head_dims(monkeypatch):
    """use_flash holds exactly on the routed head dims and even N; the kernels take every head dim in
    KERNEL_HEAD_DIMS and refuse the others."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    monkeypatch.setattr(co, "FLASH_ATTENTION", True)
    assert KERNEL_HEAD_DIMS == {hd for hd in range(32, 161, 8) if hd not in (56, 120, 152)}
    for N in (196, 256, 576):
        for hd in range(1, 200):
            assert co.use_flash(N, hd) == (hd in ROUTED), (N, hd)
    for hd in (16, 24, 56, 76, 120, 152, 168):
        assert not co.use_flash(256, hd), hd
    for N in (197, 257, 577):
        for hd in sorted(KERNEL_HEAD_DIMS):
            assert not co.use_flash(N, hd), (N, hd)
    monkeypatch.setattr(co, "FLASH_ATTENTION", False)
    assert not co.use_flash(256, 64)
    B, N, H = 1, 64, 1
    for hd in range(8, 177, 8):
        qkv = torch.zeros(B * N, 3 * H * hd, device="cuda", dtype=torch.bfloat16)
        out = torch.empty(B * N, H * hd, device="cuda", dtype=torch.bfloat16)
        if hd in KERNEL_HEAD_DIMS:
            co._C.attention_fwd(qkv, out, None, None, B, N, H, hd)
        else:
            with pytest.raises(RuntimeError):
                co._C.attention_fwd(qkv, out, None, None, B, N, H, hd)
