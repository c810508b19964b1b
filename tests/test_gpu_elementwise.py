"""Memory-bound sm_90a kernels vs the fp32 PyTorch reference ops."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _mods():
    from vit_10b_fsdp_example_b200.ops import cuda_ops, torch_ops

    return cuda_ops, torch_ops


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(torch.bfloat16)


def _close(got, ref, rel=2e-2):
    """Per-element relative + absolute bound (tests/helpers.py), not a max-normalised one."""
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel)


@pytest.mark.parametrize("rows,D", [(300, 192), (257, 1024), (512, 5120)])
def test_layernorm(rows, D):
    co, to = _mods()
    x, w, b = _rand(rows, D) * 2 + 0.5, _rand(D), _rand(D)
    y, mean, rstd = co.ln_fwd(x, w, b, 1e-5)
    yr, meanr, rstdr = to.ln_fwd(x.float(), w.float(), b.float(), 1e-5)
    _close(y, yr)
    _close(mean, meanr, rel=1e-3)
    _close(rstd, rstdr, rel=1e-3)
    dy, dres = _rand(rows, D), _rand(rows, D)
    dx, dw, db, dxs = co.ln_bwd(dy, x, w, mean, rstd, dres=dres, want_dxsum=True)
    dxr, dwr, dbr, dxsr = to.ln_bwd(dy.float(), x.float(), w.float(), meanr, rstdr, dres=dres.float(), want_dxsum=True)
    _close(dx, dxr)
    _close(dw, dwr)
    _close(db, dbr)
    _close(dxs, dxsr, rel=3e-2)


@pytest.mark.parametrize("rows,D,res,dxsum", [(1000, 5120, False, True), (777, 5120, True, False), (600, 4096, True, True),
                                              (300, 2560, False, False), (4096, 5120, True, True)])
def test_layernorm_bwd_stream(rows, D, res, dxsum):
    """Wide-row backward (csrc/layernorm_stream.cu: cp.async.bulk row ring, register column sums): every combination
    of residual-gradient input / dx column sums, row counts that do and do not divide by the SM count."""
    co, to = _mods()
    x, w, b = _rand(rows, D) * 1.5 + 3.0, _rand(D), _rand(D)   # |mean| >> std on purpose
    _, mean, rstd = co.ln_fwd(x, w, b, 1e-5)
    dy = _rand(rows, D)
    dres = _rand(rows, D) if res else None
    dx, dw, db, dxs = co.ln_bwd(dy, x, w, mean, rstd, dres=dres, want_dxsum=dxsum)
    dxr, dwr, dbr, dxsr = to.ln_bwd(dy.float(), x.float(), w.float(), mean, rstd,
                                    dres=dres.float() if res else None, want_dxsum=dxsum)
    _close(dx, dxr)
    _close(dw, dwr)
    _close(db, dbr)
    if dxsum:
        _close(dxs, dxsr, rel=3e-2)
    else:
        assert dxs is None


@pytest.mark.parametrize("n,ld", [(256, 256), (196, 200), (576, 576), (64, 64)])
def test_softmax(n, ld):
    co, _ = _mods()
    rows = 1000
    s = _rand(rows, ld) * 3
    ref = torch.softmax(s[:, :n].float() * 0.125, dim=-1)
    p = s.clone()
    co._C.softmax_fwd(p, rows, n, ld, 0.125)
    _close(p[:, :n], ref)
    dp = _rand(rows, ld)
    pr = p[:, :n].float()
    dsr = 0.125 * pr * (dp[:, :n].float() - (dp[:, :n].float() * pr).sum(-1, keepdim=True))
    d = dp.clone()
    co._C.softmax_bwd(d, p, rows, n, ld, 0.125)
    _close(d[:, :n], dsr)


def test_cross_entropy():
    co, to = _mods()
    logits = _rand(128, 1000) * 3
    target = torch.randint(0, 1000, (128,), device="cuda")
    loss, dl, correct = co.cross_entropy(logits, target)
    lossr, dlr, correctr = to.cross_entropy(logits.float(), target)
    assert abs(loss.item() - lossr.item()) < 1e-3 * abs(lossr.item())
    _close(dl, dlr)
    assert int(correct.item()) == int(correctr.item())


def test_im2col_colsum_sumsq():
    co, to = _mods()
    img = torch.randn(4, 3, 224, 224, device="cuda")
    cols = co.patch_im2col(img, 14, 640, torch.bfloat16)
    colsr = to.patch_im2col(img, 14, 640, torch.bfloat16)
    assert torch.equal(cols, colsr)
    x = _rand(3000, 1024)
    _close(co.colsum(x), x.float().sum(0), rel=1e-3)
    out = torch.zeros(1, device="cuda")
    co.sumsq(x, out)
    assert abs(out.item() - x.float().pow(2).sum().item()) < 1e-3 * out.item()


def test_adamw_split_matches_fp32_reference():
    co, to = _mods()
    n = 100_003
    w = torch.randn(n, device="cuda") * 0.02
    hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty(n, dtype=torch.int16, device="cuda")
    co.split_fp32(w, hi, lo)
    back = torch.empty_like(w)
    co.merge_fp32(hi, lo, back)
    assert torch.equal(back, w)                      # the split representation is exact
    assert (hi.float() - w).abs().max() <= (w.abs().max() * 2 ** -8)  # `hi` is the nearest bf16
    assert (hi != w.to(torch.bfloat16)).float().mean() < 1e-3        # == RN-even cast except on exact ties
    m, v = torch.zeros_like(w), torch.zeros_like(w)
    wr, mr, vr = w.clone(), m.clone(), v.clone()
    clip = torch.tensor([0.5], device="cuda")
    for step in range(1, 4):
        g = torch.randn(n, device="cuda")
        co.adamw_split(hi, lo, m, v, g, clip, 1e-3, 0.9, 0.999, 1e-8, 0.1, step)
        to.adamw_fp32(wr, mr, vr, g, clip, 1e-3, 0.9, 0.999, 1e-8, 0.1, step)
    co.merge_fp32(hi, lo, back)
    assert (back - wr).abs().max().item() < 1e-6
    assert (hi != back.to(torch.bfloat16)).float().mean() < 1e-3
    # fp32-master flavour
    w2, m2, v2 = w.clone(), torch.zeros_like(w), torch.zeros_like(w)
    wr2, mr2, vr2 = w.clone(), torch.zeros_like(w), torch.zeros_like(w)
    g = torch.randn(n, device="cuda").to(torch.bfloat16)
    co.adamw_fp32(w2, m2, v2, g, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1)
    to.adamw_fp32(wr2, mr2, vr2, g, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1)
    assert (w2 - wr2).abs().max().item() < 1e-6
