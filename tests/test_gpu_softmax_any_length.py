"""Row softmax forward / backward kernels (csrc/elementwise.cu) at row lengths the bf16x2 pair kernels do not take: odd n
(odd patch grids: 7 x 7, 15 x 15, 37 x 37 tokens) and n > 1024 (long grids), against fp32 torch.  The padding columns
n..ld-1 hold a NaN sentinel: a kernel that read them as scores would spread the NaN, one that wrote them would change
its bits."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

SCALE = 0.125


def _pad8(n):
    return (n + 7) // 8 * 8


def _close(got, ref, rel=2e-2, what=""):
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel, what=what)


def _with_sentinel(x, n):
    x = x.clone()
    x[:, n:] = float("nan")
    return x


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("n", [1, 3, 49, 225, 1023, 1025, 1156, 1369, 1764, 4096])
def test_softmax_any_row_length(n):
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    rows, ld = 300, _pad8(n)
    g = torch.Generator(device="cuda").manual_seed(n)
    s = torch.randn(rows, ld, device="cuda", generator=g) * 3
    s[::7] *= 100   # large score magnitudes: rows far from the exp range, nearly one-hot after the softmax
    s[1::7] -= 1e4  # a large common offset
    s = _with_sentinel(s.to(torch.bfloat16), n)
    ref = torch.softmax(s[:, :n].float() * SCALE, dim=-1)
    p = s.clone()
    co._C.softmax_fwd(p, rows, n, ld, SCALE)
    _close(p[:, :n], ref, what="P")
    assert _same_bits(p[:, n:], s[:, n:]), "padding columns written"

    dp = _with_sentinel((torch.randn(rows, ld, device="cuda", generator=g)).to(torch.bfloat16), n)
    pr, dpr = p[:, :n].float(), dp[:, :n].float()
    dsr = SCALE * pr * (dpr - (dpr * pr).sum(-1, keepdim=True))
    d = dp.clone()
    co._C.softmax_bwd(d, p, rows, n, ld, SCALE)
    _close(d[:, :n], dsr, what="dS")
    assert _same_bits(d[:, n:], dp[:, n:]), "padding columns written"


def test_softmax_rejects_bad_shapes():
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    x = torch.zeros(4, 64, device="cuda", dtype=torch.bfloat16)
    for n, ld, msg in [(0, 64, "n must be >= 1"), (65, 64, "ld must be >= row length"),
                       (49, 52, "multiple of 8"), (62, 63, "ld must be even")]:
        with pytest.raises(RuntimeError, match=msg):
            co._C.softmax_fwd(x, 2, n, ld, SCALE)
        with pytest.raises(RuntimeError, match=msg):
            co._C.softmax_bwd(x, x, 2, n, ld, SCALE)
