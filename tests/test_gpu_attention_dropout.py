"""Attention dropout inside the fused attention kernels (csrc/attention_drop_sm90.cu).

The mask must be exactly the one the stand-alone Philox dropout kernel draws for the un-fused path's [B*H, N, ldp]
probability buffer, so the reference mask is always co.dropout(ones[B*H, N, ldp], p, key) != 0, cut to [..., :N]."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

KEY = 0x1234_5678_9ABC_DEF


def _ref_mask(co, B, N, H, p, key):
    ldp = (N + 7) // 8 * 8
    ones = torch.ones(B * H, N, ldp, device="cuda", dtype=torch.bfloat16)
    return (co.dropout(ones, p, key) != 0)[..., :N].reshape(B, H, N, N)


def _scale(p):
    thresh = int(p * 65536.0 + 0.5)
    return 1.0 / (1.0 - thresh / 65536.0)


def _heads(t, B, N, H, hd, parts):
    """[B*N, parts*H*hd] -> [parts, B, H, N, hd]"""
    return t.float().view(B, N, parts, H, hd).permute(2, 0, 3, 1, 4)


def _pack(q, k, v):
    """[B, H, N, hd] x 3 -> packed qkv [B*N, 3*H*hd] bf16"""
    B, H, N, hd = q.shape
    return torch.stack([q, k, v], 0).permute(1, 3, 0, 2, 4).reshape(B * N, 3 * H * hd).to(torch.bfloat16).contiguous()


def _eye_rows(B, H, N, hd):
    e = torch.zeros(B, H, N, hd, device="cuda")
    e[..., torch.arange(N), torch.arange(N)] = 1.0
    return e


def _run(co, qkv, dout, B, N, H, hd, drop):
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd, drop=drop)
    dqkv = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, drop=drop)
    return out, lse, dqkv


# ---- 1. exact mask readouts (Q = K = 0 -> uniform P; N <= hd so one-hot rows fit) ----
@pytest.mark.parametrize("B,N,H,hd", [(2, 100, 2, 128), (1, 64, 3, 64), (1, 160, 2, 160), (2, 100, 1, 160)])
def test_forward_and_dv_read_out_the_mask(B, N, H, hd):
    """O = (P o M s) V with V rows one-hot gives O[q, j] = s / N * M[q, j]; dV = (P o M s)^T dO with dO rows one-hot
    gives dV[k, j] = s / N * M[j, k]."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    p = 0.3
    zeros = torch.zeros(B, H, N, hd, device="cuda")
    eye = _eye_rows(B, H, N, hd)
    qkv = _pack(zeros, zeros, eye)
    dout = eye.permute(0, 2, 1, 3).reshape(B * N, H * hd).to(torch.bfloat16)
    m = _ref_mask(co, B, N, H, p, KEY)
    out, _, dqkv = _run(co, qkv, dout, B, N, H, hd, (p, KEY))
    o = _heads(out, B, N, H, hd, 1)[0][..., :N]
    assert torch.equal(o != 0, m)
    kept = o[m]
    assert torch.allclose(kept, torch.full_like(kept, _scale(p) / N), rtol=1e-2)
    dv = _heads(dqkv, B, N, H, hd, 3)[2][..., :N]
    assert torch.equal(dv != 0, m.transpose(-1, -2))


@pytest.mark.parametrize("B,N,H,hd", [(2, 100, 2, 128), (1, 64, 3, 64), (1, 160, 2, 160)])
@pytest.mark.parametrize("role", ["dq", "dk"])
def test_dq_dk_signs_read_out_the_mask(B, N, H, hd, role):
    """All V rows = v, all dO rows = w (w.v = c > 0), p = 0.5: dP = c, delta_q = c s r_q with r_q the kept fraction of
    row q, so dS[q, k] = P s c * scale * (M[q, k] - r_q) has the sign of 2 M - 1.  K one-hot rows (Q = 0) read dS out
    through dQ = dS K; Q one-hot rows (K = 0) read dS^T out through dK = dS^T Q."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    p = 0.5
    zeros = torch.zeros(B, H, N, hd, device="cuda")
    eye = _eye_rows(B, H, N, hd)
    ones = torch.ones(B, H, N, hd, device="cuda")
    qkv = _pack(zeros, eye, ones) if role == "dq" else _pack(eye, zeros, ones)
    dout = torch.ones(B * N, H * hd, device="cuda", dtype=torch.bfloat16)
    m = _ref_mask(co, B, N, H, p, KEY)
    r = m.float().mean(dim=-1)
    assert ((r > 0) & (r < 1)).all()
    _, _, dqkv = _run(co, qkv, dout, B, N, H, hd, (p, KEY))
    g = _heads(dqkv, B, N, H, hd, 3)
    if role == "dq":
        got = g[0][..., :N]
        assert torch.equal(got > 0, m) and torch.equal(got < 0, ~m)
    else:
        got = g[1][..., :N]
        assert torch.equal(got > 0, m.transpose(-1, -2)) and torch.equal(got < 0, ~m.transpose(-1, -2))


# ---- 2. numerics ----
def _reference(qkv, dout, B, N, H, hd, m, p):
    q, k, v = _heads(qkv, B, N, H, hd, 3)
    do = _heads(dout, B, N, H, hd, 1)[0]
    ms = m.float() * _scale(p)
    P = torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1)
    o = (P * ms) @ v
    dv = (P * ms).transpose(-1, -2) @ do
    delta = (do * o).sum(-1, keepdim=True)
    ds = hd ** -0.5 * P * ((do @ v.transpose(-1, -2)) * ms - delta)
    dq, dk = ds @ k, ds.transpose(-1, -2) @ q
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * N, H * hd)  # noqa: E731
    dqkv = torch.cat([flat(dq), flat(dk), flat(dv)], dim=1)
    return flat(o), dqkv


def _close_max(got, ref, what, rel=3e-2):
    err = (got.float() - ref.float()).abs().max().item() / (ref.float().abs().max().item() + 1e-6)
    assert err < rel, f"{what}: rel err {err}"


@pytest.mark.parametrize("B,N,H,hd", [(2, 256, 4, 160), (3, 196, 3, 64), (2, 128, 2, 128), (1, 576, 2, 160)])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_fused_dropout_matches_references(B, N, H, hd, p):
    from helpers import assert_close_elementwise
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + N + hd)
    qkv = (torch.randn(B * N, 3 * D, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    drop = (p, KEY)
    out, lse = co.attention_fwd_lse(qkv, B, N, H, hd, drop=drop)
    n0 = co.launch_count()
    dqkv, cs = co.attention_bwd_lse(dout, qkv, out, lse, B, N, H, hd, want_colsum=True, drop=drop)
    assert co.launch_count() - n0 == 1
    # fp32 reference with the exact mask
    m = _ref_mask(co, B, N, H, p, KEY)
    outr, dqkvr = _reference(qkv, dout, B, N, H, hd, m, p)
    assert_close_elementwise(out, outr, rtol=3e-2, atol_rel=3e-2, what="out")
    q, k, _ = _heads(qkv, B, N, H, hd, 3)
    lser = torch.logsumexp((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1).reshape(B * H, N)
    assert (lse - lser).abs().max().item() < 2e-2  # log-sum-exp of the undropped scores
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        _close_max(dqkv[:, sl], dqkvr[:, sl], name)
    assert_close_elementwise(cs, dqkvr.sum(0), rtol=5e-2, atol_rel=5e-2, what="qkv bias grad")
    # today's un-fused GPU path (materialised P + Philox dropout kernel) with the same key
    outu, P = co.attention_fwd(qkv, B, N, H, hd, drop=drop)
    dqkvu, csu = co.attention_bwd(dout, qkv, P, B, N, H, hd, want_colsum=True, drop=drop)
    assert_close_elementwise(out, outu, rtol=3e-2, atol_rel=3e-2, what="out vs un-fused")
    for name, sl in (("dq", slice(0, D)), ("dk", slice(D, 2 * D)), ("dv", slice(2 * D, 3 * D))):
        _close_max(dqkv[:, sl], dqkvu[:, sl], name + " vs un-fused")
    assert_close_elementwise(cs, csu, rtol=5e-2, atol_rel=5e-2, what="qkv bias grad vs un-fused")


# ---- 3. determinism ----
def test_same_key_same_bits_other_key_other_bits():
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    B, N, H, hd = 2, 196, 4, 64
    qkv = (torch.randn(B * N, 3 * H * hd, device="cuda") * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, H * hd, device="cuda").to(torch.bfloat16)
    a = _run(co, qkv, dout, B, N, H, hd, (0.1, 7))
    b = _run(co, qkv, dout, B, N, H, hd, (0.1, 7))
    c = _run(co, qkv, dout, B, N, H, hd, (0.1, 8))
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y)
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[2], c[2])
    # the forward without the log-sum-exp (first pass of a checkpointed block) gives the same output
    out, P = co.attention_fwd(qkv, B, N, H, hd, drop=(0.1, 7), need_p=False)
    assert P is None and torch.equal(out, a[0])


# ---- 4. model level ----
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=2, mlp_ratio=4.0, num_classes=96,
             att_dropout=0.1)
    d.update(kw)
    return ViTConfig(**d)


def _grads(model):
    return {u.name: u.shard_grad.float().clone() for u in model.all_units}


def _model_grads(cfg, **kw):
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=g).cuda()
    y = torch.randint(0, cfg.num_classes, (4,), generator=g).cuda()
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=4, **kw)
    loss = model.forward_backward(x, y).item()
    return loss, _grads(model)


def _agree(a, b, tol):
    (la, ga), (lb, gb) = a, b
    assert abs(la - lb) < 2e-3, (la, lb)
    for k in ga:
        assert (ga[k] - gb[k]).norm().item() <= tol * ga[k].norm().item() + 1e-6, k


@pytest.mark.parametrize("kw", [dict(), dict(embed_dim=320, num_heads=2)])
def test_model_flash_and_unfused_dropout_agree(kw, monkeypatch):
    """Same masks on both routes: gradients with the fused pair match the un-fused route (hd 64 and 160)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    cfg = _cfg(**kw)
    monkeypatch.setattr(co, "FLASH_ATTENTION", False)
    ref = _model_grads(cfg)
    monkeypatch.setattr(co, "FLASH_ATTENTION", True)
    _agree(ref, _model_grads(cfg), 3e-2)


def test_model_checkpointed_and_kept_blocks_agree():
    """The non-saving first pass, the recompute and the saving forward all apply the same mask: bitwise the same
    attention, so only GEMM accumulation order can differ."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    assert co.FLASH_ATTENTION
    cfg = _cfg()
    base = _model_grads(cfg, grad_ckpt=True, ckpt_keep_blocks=0)
    for kw in (dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        _agree(base, _model_grads(cfg, **kw), 2e-2)


def test_block_peak_memory_drops_with_fused_dropout(monkeypatch):
    """One block's forward (saving) + backward: the fused route never allocates a [B*H, N, ldp] probability buffer."""
    from vit_10b_fsdp_example_b200.models import vit
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    cfg = _cfg(embed_dim=512, num_heads=8)
    B, N, D = 16, cfg.num_patches, cfg.embed_dim
    gen = torch.Generator().manual_seed(0)
    p = {k: v.to("cuda", torch.bfloat16) for k, v in vit.init_block_params(cfg, gen).items()}
    G = {k: torch.empty_like(v) for k, v in p.items()}
    x = torch.randn(B * N, D, device="cuda").to(torch.bfloat16)
    dy = torch.randn(B * N, D, device="cuda").to(torch.bfloat16)
    dy_cs = dy.float().sum(0)
    drop = vit.DropoutCtx(seed=3)
    peaks, grads = {}, {}
    for flash in (False, True):
        monkeypatch.setattr(co, "FLASH_ATTENTION", flash)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _, s = vit.block_forward(co, cfg, p, x, B, save=True, drop=drop)
        dx, _ = vit.block_backward(co, cfg, p, G, s, dy, dy_cs, B)
        torch.cuda.synchronize()
        peaks[flash] = torch.cuda.max_memory_allocated() - base
        grads[flash] = {k: v.float().clone() for k, v in G.items()}
        del s, dx
    buf = B * cfg.num_heads * N * ((N + 7) // 8 * 8) * 2
    assert peaks[False] - peaks[True] >= buf, (peaks, buf)
    for k in grads[False]:
        a, b = grads[False][k], grads[True][k]
        assert (a - b).norm().item() <= 3e-2 * a.norm().item() + 1e-6, k
