"""Stochastic depth on the GPU: the per-sample Philox scales, the GEMM epilogue row scale, drop_path_bwd and the model.

The NumPy Philox of torch_ops is the reference for the mask bits; the fp32 torch ops are the reference for the math."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)


@pytest.mark.parametrize("key,p,B,offset", [(0x1234_5678_9ABC_DEF, 0.1, 128, 0), (7, 0.5, 1, 3),
                                            (2 ** 62 + 5, 0.3, 37, 13), (99, 0.9, 1000, 4096), (123, 0.0, 16, 0),
                                            (0x7FFF_FFFF_FFFF_FFFF, 0.25, 8, 2 ** 33)])
def test_drop_path_scale_bits_equal_the_numpy_reference(key, p, B, offset):
    from vit_10b_fsdp_example_b200.ops import torch_ops

    got = _co().drop_path_scale(key, p, B, offset, "cuda").cpu()
    ref = torch_ops.drop_path_scale(key, p, B, offset, "cpu")
    assert torch.equal(got, ref), (got, ref)


def _gemm(a, w, M, N, K, block_n, cluster, bias=None, residual=None, row_scale=None, rps=0):
    co = _co()
    d = torch.full((M, N), 3.0, device="cuda", dtype=torch.bfloat16)
    co.gemm_raw(a, K, 0, w, K, 0, d, N, M, N, K, bias=bias, residual=residual, ld_res=N if residual is not None else 0,
                block_n=block_n, cluster=cluster, row_scale=row_scale, rows_per_scale=rps)
    return d


@pytest.mark.parametrize("with_residual", [True, False])
@pytest.mark.parametrize("rps", [196, 257])
@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("block_n", [128, 256])
def test_gemm_row_scale(block_n, cluster, rps, with_residual):
    """M = 5 * rps (980 or 1285 rows: not a multiple of 128, samples straddle m-tiles)."""
    B, N, K = 5, 384, 320
    M = B * rps
    g = torch.Generator(device="cuda").manual_seed(rps + block_n + cluster)
    a = (torch.randn(M, K, device="cuda", generator=g)).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    bias = _rand(N, scale=0.5)
    res = _rand(M, N) if with_residual else None
    plain = _gemm(a, w, M, N, K, block_n, cluster, bias=bias, residual=res)
    ones = torch.ones(B, device="cuda")
    assert torch.equal(_gemm(a, w, M, N, K, block_n, cluster, bias=bias, residual=res, row_scale=ones, rps=rps), plain)

    s = torch.tensor([0.0, 1.25, 1.25, 0.0, 1.25], device="cuda")
    out = _gemm(a, w, M, N, K, block_n, cluster, bias=bias, residual=res, row_scale=s, rps=rps)
    srow = s.repeat_interleave(rps)
    ref = (a.float() @ w.float().t() + bias.float()) * srow[:, None]
    if with_residual:
        ref = ref + res.float()
    dropped = srow == 0
    if with_residual:
        assert torch.equal(out[dropped], res[dropped])
    else:
        assert torch.equal(out[dropped], torch.zeros_like(out[dropped]))
    kept = ~dropped
    err = (out[kept].float() - ref[kept]).abs()
    assert (err <= 1e-2 * ref[kept].abs() + 2e-2).all(), err.max().item()


def test_gemm_row_scale_rejects_unsupported_epilogues():
    co = _co()
    a, w = _rand(256, 128), _rand(256, 128)
    d = torch.empty(256, 256, device="cuda", dtype=torch.bfloat16)
    s = torch.ones(2, device="cuda")
    with pytest.raises(RuntimeError, match="row_scale"):
        co.gemm_raw(a, 128, 0, w, 128, 0, d, 256, 256, 256, 128, act=co.ACT_GELU, row_scale=s, rows_per_scale=128)
    with pytest.raises(RuntimeError, match="row_scale"):
        co.gemm_raw(a, 128, 0, w, 128, 0, d, 256, 256, 256, 128, colsum=torch.zeros(256, device="cuda"),
                    row_scale=s, rows_per_scale=128)


@pytest.mark.parametrize("B,N,C", [(5, 196, 640), (3, 257, 1288), (8, 256, 5120), (1, 1, 8)])
def test_drop_path_bwd(B, N, C):
    dy = _rand(B * N, C)
    s = torch.tensor([1.25 if b % 3 else 0.0 for b in range(B)], device="cuda")
    dt, cs = _co().drop_path_bwd(dy, s, N)
    ref = (dy.float() * s.repeat_interleave(N)[:, None]).bfloat16()
    assert torch.equal(dt, ref)
    csr = ref.double().sum(0)
    assert (cs.double() - csr).abs().max().item() <= 1e-5 * ref.float().abs().sum(0).max().item() + 1e-6


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             drop_path_rate=0.5)
    d.update(kw)
    return ViTConfig(**d)


def _data(B=8):
    g = torch.Generator().manual_seed(0)
    return torch.randn(B, 3, 224, 224, generator=g), torch.randint(0, 96, (B,), generator=g)


def _named_grads(model):
    out = {}
    for u in model.all_units:  # world 1: the shard buffer has the full layout
        for n, v in u.layout.param_views(u.shard_grad.float()).items():
            out[f"{u.name}.{n}"] = v.detach().cpu().clone()
    return out


def test_model_matches_the_fp32_cpu_model():
    """Same parameters (host init) and the same masks (bit-identical Philox): bf16 GPU vs fp32 CPU loss and
    gradients."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    x, y = _data()
    for keep in (0, 3):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(_cfg(), device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _named_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)
    # the masks matter: without stochastic depth the loss is another one
    ref0 = FSDPViT(_cfg(drop_path_rate=0.0), device="cuda", dtype=torch.bfloat16, seed=4)
    assert abs(ref0.forward_backward(x.cuda(), y.cuda()).item() - loss) > 1e-4


@pytest.mark.parametrize("kw", [dict(), dict(mlp_dropout=0.1)])
def test_checkpointed_and_kept_blocks_give_the_same_gradients(kw):
    """The recompute regenerates the same scale vectors: every GEMM-produced weight gradient is bitwise equal.  Biases
    and LayerNorm parameters are column sums reduced with fp32 atomics in arrival order, and so is the loss; the last
    fp32 bits of those vary from run to run, which can flip the rounding of the bf16 gradient buffer by one ulp."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    x, y = _data()
    runs = []
    for mkw in (dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=3),
                dict(grad_ckpt=False)):
        model = FSDPViT(_cfg(**kw), device="cuda", dtype=torch.bfloat16, seed=4, **mkw)
        runs.append((model.forward_backward(x.cuda(), y.cuda()).item(), _named_grads(model)))
    (l0, g0) = runs[0]
    for l1, g1 in runs[1:]:
        assert abs(l0 - l1) <= 1e-6 * abs(l0), (l0, l1)
        for k in g0:
            linear_weight = k.endswith(("qkv.weight", "proj.weight", "fc1.weight", "fc2.weight", "head.weight"))
            diff = (g0[k] - g1[k]).abs().max().item()
            if linear_weight:
                assert torch.equal(g0[k], g1[k]), (k, diff, g0[k].abs().max().item())
            else:
                one_ulp = g0[k].abs() * 2.0 ** -7 + 1e-6 * g0[k].abs().max().item()  # bf16: 8 significant bits
                assert ((g0[k] - g1[k]).abs() <= one_ulp).all(), (k, diff, g0[k].abs().max().item())
