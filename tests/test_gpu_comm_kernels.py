"""The NVLink collective kernels (csrc/comm.cu) and the all-gather fused into the GEMM (csrc/gemm_sm90.cu), on one GPU,
against exact and float64 references.

A peer of these kernels is nothing but a raw device pointer, so W separate allocations on one device stand in for the
W ranks ("virtual peers"):
  * reduce_scatter with an empty sync list runs no flag protocol (to_sync gives world 1), yet it still reduces over
    all W pointers it is given;
  * p2p_all_gather has no flags at all;
  * the fused GEMM's gather uses only its local counters (ag.flags).
All three are plain stream-ordered launches.  The segment tables and the fusion spec come from the real
Sm100Backend._ag_table / _rs_table / ag_fuse_spec, called on a stand-in backend object that carries the extension's
chunk sizes, so the host tables and the kernels are tested together.  W runs over 2, 3, 5, 8 and 16 (the kernels'
kMaxWorld), the rank over 0, a middle rank and W - 1 (the staggered source order and the GEMM's n-tile rotation), and
max_ctas over 1, 3, 0 (the default 64) and 132, so CTAs walk many segments in their grid-stride loops.

Not tested here, because a peer's flags would have to be pre-seeded and a wrong seed spins into the kernels' trap: the
NVLS multimem paths, the cross-GPU flag protocol (sync_begin / sync_end), all_reduce_mean, signal_barrier and
allreduce_scalars.  They stay with tests/test_gpu_multi.py and tests/test_flag_protocol_model.py.

The CPU meta-tests at the end show that the references agree with plain numpy and that every checker rejects a
specific wrong kernel.

Run as a script (``python tests/test_gpu_comm_kernels.py no_l2_hint``) it checks the pull all-gather with
B200_COMM_L2_HINT=0, which the extension reads once per process.
"""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from helpers import assert_close_elementwise  # noqa: E402
from test_gpu_memory_bound_fp64 import (FLT_MIN, U, _f32, adamw_state, assert_within, check_adamw,  # noqa: E402
                                        check_split, gelu_ref)
from vit_10b_fsdp_example_b200.config import ViTConfig  # noqa: E402
from vit_10b_fsdp_example_b200.models import vit  # noqa: E402
from vit_10b_fsdp_example_b200.parallel.backends import Sm100Backend  # noqa: E402
from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout  # noqa: E402

WORLDS = (2, 3, 5, 8, 16)
MAX_CTAS = (1, 3, 0, 132)
VITL = ViTConfig(embed_dim=1024, num_heads=16, num_blocks=24, patch_size=16)
VIT10B = ViTConfig()
# Segments shorter than one chunk (a 64-element group is 128 bytes; an all-gather chunk is 16 KiB, a reduce-scatter chunk
# 512 16-byte vectors) and segments that end mid-chunk (the 9 x 4099 group).  The 240-row weight is a whole number of
# rows per rank at every W; at W = 2, 3 and 5 it is also a whole number of 64-element blocks, so fusable_params takes it.
SYNTH = [("norm1.weight", (37,)), ("attn.qkv.weight", (240, 24)), ("attn.qkv.bias", (3, 50)), ("tiny", (8,)),
         ("mlp.fc1.weight", (9, 4099)), ("mlp.fc1.bias", (1000,))]
KINDS = ("vitl_block", "vitl_block_flat", "synthetic", "vit10b_root")
CASES = [(k, w) for k in KINDS[:3] for w in WORLDS] + [("vit10b_root", 8)]
DTYPES = {"bf16": torch.bfloat16, "fp32": torch.float32}


def unit_layout(kind, world):
    """ViT-L block (per-parameter groups or one flat parameter), the small synthetic unit, or the ViT-10B root unit
    (patch embedding padded to the TMA K, position embedding, 1000-class head: 125 rows per rank at W = 8)."""
    if kind.startswith("vitl_block"):
        return UnitLayout.build("blocks.0", vit.block_param_specs(VITL), world, kind.endswith("flat"))
    if kind == "synthetic":
        return UnitLayout.build("synthetic", SYNTH, world, False)
    assert kind == "vit10b_root"
    return UnitLayout.build("root", vit.root_param_specs(VIT10B), world, False)


def virtual_backend(world, rank, device="cuda", C=None):
    """A stand-in Sm100Backend: the real table and spec builders run on it, with the extension's chunk sizes."""
    if C is None:
        from vit_10b_fsdp_example_b200.ops import native

        C = native.load()
    be = types.SimpleNamespace(world=world, rank=rank, device=device, _C=C, _seg_cache={}, _peer={},
                               FUSED_PARAMS=Sm100Backend.FUSED_PARAMS)
    be._lay_key = Sm100Backend._lay_key
    return be


def ranks(world):
    return sorted({0, world // 2, world - 1})


def seed_of(*parts):
    s = 0
    for p in parts:
        s = s * 131 + p
    return s % (2 ** 31)


def int_view(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def assert_bitwise(name, got, exp):
    """Every element has the expected bit pattern (NaN payloads and the sign of zero included)."""
    gi, ei = int_view(got), int_view(exp)
    bad = gi != ei
    if bool(bad.any()):
        i = int(bad.nonzero()[0, 0])
        w = 2 * got.element_size()
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ bitwise; first at flat index "
                             f"{i}: got {got[i].item()!r} (0x{int(gi[i]) & (16 ** w - 1):0{w}x}), expected "
                             f"{exp[i].item()!r} (0x{int(ei[i]) & (16 ** w - 1):0{w}x})")


def sentinel(n, dtype, device="cuda"):
    """A NaN bit pattern no kernel computes: whatever still holds it was not written."""
    bits = 0x7FA5 if dtype == torch.bfloat16 else 0x7FA5A5A5
    it = torch.int16 if dtype == torch.bfloat16 else torch.int32
    return torch.full((n,), bits, dtype=it, device=device).view(dtype)


# ------------------------------------------------------------------------------------------------
# reduce-scatter: the exact fp32 replay of the kernel and the float64 mean
# ------------------------------------------------------------------------------------------------
def grad_values(n, seed, dtype, device="cuda"):
    """Gradients of mixed magnitude (|g| ~ 1e-3 ... 1e3), both signs.  At indices shared by every peer: exact zeros
    (every 11th), negative zeros (every 13th from 5: all peers -0, whose sum is +0) and subnormals (every 29th from 7)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    mag = 10.0 ** (torch.rand(n, generator=gen, device=device) * 6 - 3)
    g = torch.randn(n, generator=gen, device=device) * mag
    g[::11] = 0.0
    g[5::13] = -0.0
    g[7::29] = 3e-39 * torch.sign(g[7::29] + 0.5)
    return g.to(dtype)


def ftz(x):
    """The extension is built with --use_fast_math, i.e. -ftz=true: every fp32 add and multiply flushes subnormal
    inputs and results to a zero of the same sign."""
    return torch.where(x.abs() < FLT_MIN, x * 0, x)


def rs_replay(slices, rank, order=None, scale=None):
    """What reduce_scatter_kernel computes on the peer-pull path, bit for bit: start from +0.0, add the peers in the
    order rank, rank + 1, ... mod W in fp32 (reduce_vec staggers the sources that way), then multiply by
    float32(1 / W), which is the scale Sm100Backend.reduce_scatter passes.  `order` / `scale` build the mutants."""
    W = len(slices)
    order = [(rank + k) % W for k in range(W)] if order is None else order
    acc = torch.zeros(slices[0].shape, dtype=torch.float32, device=slices[0].device)
    for p in order:
        acc = ftz(acc + ftz(slices[p].float()))
    return ftz(acc * (_f32(1.0 / W) if scale is None else scale))


def shard_slices(lay, peers, rank):
    """This rank's slices of every peer's full gradient buffer, in shard order."""
    return [lay.shard_from_full(p, rank, torch.empty(lay.shard_numel, dtype=p.dtype, device=p.device)) for p in peers]


def check_reduce_scatter(slices, rank, out):
    """Bitwise against the fp32 replay, then against the float64 mean.  The kernel's W - 1 fp32 additions (the first
    add to +0.0 is exact) each err by at most u of a partial sum, <= u sum|g|; float32(1 / W) and the product each add
    u of the result, <= u sum|g| / W; a flushed subnormal moves a value by less than FLT_MIN:
        |out - sum(g) / W| <= (W - 1) u sum|g| / W + 2 u sum|g| / W + (W + 2) FLT_MIN"""
    assert_bitwise("reduce_scatter out vs the fp32 replay", out, rs_replay(slices, rank))
    W = len(slices)
    s64 = sum(s.double() for s in slices)
    a64 = sum(s.double().abs() for s in slices)
    assert_within("reduce_scatter out vs the float64 mean", out, s64 / W, (W + 1.01) * U * a64 / W + (W + 2) * FLT_MIN)


def check_sumsq(sumsq, s0, out, chunks, grid, kvec):
    """sumsq_out accumulates with atomics, so it starts from s0 != 0.  Each thread sums the squares of its elements
    serially (at most 4 vectors of kvec elements per chunk, ceil(chunks / grid) chunks), a warp adds its 32 partials in
    5 levels, and every warp of every CTA adds its partial to sumsq_out with one fp32 atomic.  All terms are positive:
        |sumsq - (s0 + sum out^2)| <= (per_thread + 5 + 4 grid) u (s0 + sum out^2)"""
    ref = s0 + out.double().square().sum()
    per_thread = -(-chunks // grid) * 4 * kvec
    tol = (per_thread + 5 + 4 * grid) * U * ref
    assert_within("reduce_scatter sumsq_out", sumsq.reshape(1), ref.reshape(1), tol.reshape(1))


def rs_grid(chunks, max_ctas):
    return max(1, min(chunks, max_ctas if max_ctas > 0 else 64))


def run_reduce_scatter(be, lay, peers, out, sumsq, max_ctas, adam=None):
    """One reduce_scatter launch on the virtual peers, with the arguments Sm100Backend.reduce_scatter passes and no
    flag protocol.  Returns the chunk count of the table."""
    table, chunks = Sm100Backend._rs_table(be, lay, peers[0].element_size())
    a = tuple(adam) if adam is not None else (None, None, None, None, [])
    be._C.reduce_scatter([p.data_ptr() for p in peers], 0, be.rank, be.world, out, table, chunks,
                         peers[0].dtype == torch.bfloat16, 1.0 / be.world, sumsq, max_ctas, [], [], None, None, *a)
    return chunks


@pytest.mark.gpu
@pytest.mark.parametrize("dname", sorted(DTYPES))
@pytest.mark.parametrize("kind,world", CASES)
def test_reduce_scatter(kind, world, dname):
    dtype = DTYPES[dname]
    lay = unit_layout(kind, world)
    peers = [grad_values(lay.full_numel, seed_of(KINDS.index(kind), world, r, dtype.itemsize), dtype)
             for r in range(world)]
    before = [p.clone() for p in peers]
    kvec = 16 // dtype.itemsize
    for rank in ranks(world):
        be = virtual_backend(world, rank)
        slices = shard_slices(lay, peers, rank)
        for max_ctas in MAX_CTAS:
            out = sentinel(lay.shard_numel, torch.float32)
            s0 = 0.75
            sumsq = torch.full((1,), s0, device="cuda")
            chunks = run_reduce_scatter(be, lay, peers, out, sumsq, max_ctas)
            torch.cuda.synchronize()
            check_reduce_scatter(slices, rank, out)
            check_sumsq(sumsq, s0, out, chunks, rs_grid(chunks, max_ctas), kvec)
    for r, (p, b) in enumerate(zip(peers, before)):
        assert_bitwise(f"peer {r}'s gradient buffer after the reduce-scatters", p, b)


# ------------------------------------------------------------------------------------------------
# AdamW fused into the reduce-scatter
# ------------------------------------------------------------------------------------------------
def f32_ulp(x64):
    """Spacing of the fp32 numbers at each float64 value: 2^(e - 24) for |x| = m 2^e, m in [0.5, 1)."""
    _, e = torch.frexp(x64.abs().clamp_min(FLT_MIN))
    return torch.ldexp(torch.ones_like(x64), e - 24)


def check_fused_matches_split(m0, v0, g, hp, step, fused, split):
    """The fused update against adamw_split run on a copy of the same state with the same gradient.  Both evaluate the
    same fp32 expressions, except that the host hands the fused kernel an IEEE 1 / bc while adamw_split forms 1 / bc on
    the device with the approximate reciprocal (--use_fast_math), at most 2 ulp apart.  m and v are the same
    expressions of the same inputs, but the two kernels may contract b1 m0 + (1 - b1) g into an fma differently: 2 u of
    their terms.  Where m cancels that is most of m, so the update is measured, as in check_adamw, by
    lr (b1 |m0| + (1 - b1) |g|) / bc1 / (sqrt(v / bc2) + eps).  Against that, the numerator moves by 2 u for m, 3 u for
    the reciprocal and 1 u for its own rounding; the denominator's v / bc2 by 4 u (2 u after the square root) plus 1 u
    each for the square root and the eps add; then 2 u for the approximate divide and 1 u for the lr product: 14 u,
    taken as 16 u.  The new w = w0 decay - update is rounded once in each kernel, so the two may be one fp32 ulp of w
    apart beyond that:
        |w_fused - w_split| <= 16 u |update| + ulp(w_split)"""
    lr, b1, b2, eps, _ = hp
    (w, m, v), (w2, m2, v2) = fused, split
    gd = g.double()
    m_terms = b1 * m0.double().abs() + (1 - b1) * gd.abs()
    assert_within("fused AdamW m vs adamw_split", m, m2.double(), 2 * U * m_terms)
    assert_within("fused AdamW v vs adamw_split", v, v2.double(), 2 * U * (b2 * v0.double() + (1 - b2) * gd * gd))
    upd = (lr / (1 - b1 ** step)) * m_terms / ((v2.double() / (1 - b2 ** step)).sqrt() + eps)
    assert_within("fused AdamW w vs adamw_split", w, w2.double(), 16 * U * upd + f32_ulp(w2.double()))


ADAM_STEPS = [1, 2, 3, 10, 1000, 10000]
# (layout, W, rank, max_ctas)
ADAM_CASES = [("synthetic", 5, 2, 3), ("vitl_block", 8, 7, 0), ("vit10b_root", 8, 0, 132)]


@pytest.mark.gpu
@pytest.mark.parametrize("step", ADAM_STEPS)
def test_adamw_fused_into_reduce_scatter(step):
    """kAdam: the reduced gradient goes straight into the sharded AdamW update of the split master.  Its hyper list is
    [lr, beta1, beta2, eps, wd, step] as ShardedAdamW.fused_args passes it; the state comes from adamw_state (exact bf16
    ties, weights that cross zero, zero moments at step 1)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    hyper = [1e-3, 0.9, 0.999, 1e-8, 0.1, float(step)]
    hp = tuple(_f32(t) for t in hyper[:5])
    for kind, world, rank, max_ctas in ADAM_CASES:
        lay = unit_layout(kind, world)
        n = lay.shard_numel
        peers = [grad_values(lay.full_numel, seed_of(step, world, r), torch.bfloat16) for r in range(world)]
        be = virtual_backend(world, rank)
        gmean = rs_replay(shard_slices(lay, peers, rank), rank)
        w0, m0, v0 = adamw_state(n, step, seed=seed_of(step, world))
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        lo = torch.empty(n, dtype=torch.int16, device="cuda")
        co.split_fp32(w0, hi, lo)
        m, v = m0.clone(), v0.clone()
        out = sentinel(n, torch.float32)
        sumsq = torch.full((1,), 0.5, device="cuda")
        chunks = run_reduce_scatter(be, lay, peers, out, sumsq, max_ctas, adam=(hi, lo, m, v, hyper))
        w = torch.empty_like(w0)
        co.merge_fp32(hi, lo, w)
        torch.cuda.synchronize()
        assert_bitwise("out in fused mode (must not be written)", out, sentinel(n, torch.float32))
        check_split(hi, lo, w)
        check_adamw(w0, m0, v0, gmean, 1.0, hp, step, w, m, v)
        check_sumsq(sumsq, 0.5, gmean, chunks, rs_grid(chunks, max_ctas), 8)
        # the stand-alone path: unfused reduce-scatter, then adamw_split on a copy of the same state
        g = sentinel(n, torch.float32)
        run_reduce_scatter(be, lay, peers, g, None, max_ctas)
        hi2, lo2 = torch.empty_like(hi), torch.empty_like(lo)
        co.split_fp32(w0, hi2, lo2)
        m2, v2 = m0.clone(), v0.clone()
        co.adamw_split(hi2, lo2, m2, v2, g, None, *hp, step)
        w2 = torch.empty_like(w0)
        co.merge_fp32(hi2, lo2, w2)
        torch.cuda.synchronize()
        assert_bitwise("unfused reduce-scatter vs the fp32 replay", g, gmean)
        check_fused_matches_split(m0, v0, gmean, hp, step, (w, m, v), (w2, m2, v2))


# ------------------------------------------------------------------------------------------------
# pull all-gather
# ------------------------------------------------------------------------------------------------
def random_bits(n, dtype, seed, device="cuda"):
    """Uniformly random bit patterns, plus explicit quiet, signalling and negative NaN encodings every 101st element."""
    it = torch.int16 if dtype == torch.bfloat16 else torch.int32
    info = torch.iinfo(it)
    gen = torch.Generator(device=device).manual_seed(seed)
    bits = torch.randint(info.min, info.max, (n,), generator=gen, device=device, dtype=it)
    nans = (0x7FC1, 0x7F81, -1) if it == torch.int16 else (0x7FC00001, 0x7F800001, -1)
    for k, nan in enumerate(nans):
        bits[37 * k::101] = nan
    return bits.view(dtype)


def check_all_gather(lay, full_ref, out, exclude):
    """out is layout.full_from_shards byte for byte, except that the excluded groups (gathered later by the GEMM that
    consumes them) still hold the sentinel."""
    exp = full_ref.clone()
    for g in lay.groups:
        if g.name in exclude:
            exp[g.full_offset: g.full_offset + lay.world * g.shard_len] = sentinel(lay.world * g.shard_len, exp.dtype,
                                                                                   exp.device)
    assert_bitwise(f"p2p_all_gather (exclude {sorted(exclude)})", out, exp)


def run_all_gather_case(kind, world, dtype):
    """Every rank of `ranks(world)` at every max_ctas, alternating between no exclusion and the backend's
    fusable_params."""
    lay = unit_layout(kind, world)
    shards = [random_bits(lay.shard_numel, dtype, seed_of(KINDS.index(kind), world, r, dtype.itemsize))
              for r in range(world)]
    before = [s.clone() for s in shards]
    full_ref = lay.full_from_shards(shards, torch.empty(lay.full_numel, dtype=dtype, device="cuda"))
    n_excluded = 0
    for i, rank in enumerate(ranks(world)):
        be = virtual_backend(world, rank)
        fusable = Sm100Backend.fusable_params(be, lay)
        for j, max_ctas in enumerate(MAX_CTAS):
            exclude = fusable if (i + j) % 2 else ()
            n_excluded += len(exclude)
            table, chunks = Sm100Backend._ag_table(be, lay, dtype.itemsize, exclude)
            out = sentinel(lay.full_numel, dtype)
            be._C.p2p_all_gather([s.data_ptr() for s in shards], rank, out, table, chunks, max_ctas)
            torch.cuda.synchronize()
            check_all_gather(lay, full_ref, out, exclude)
    for r, (s, b) in enumerate(zip(shards, before)):
        assert_bitwise(f"rank {r}'s shard after the all-gathers", s, b)
    return n_excluded


@pytest.mark.gpu
@pytest.mark.parametrize("dname", sorted(DTYPES))
@pytest.mark.parametrize("kind,world", CASES)
def test_pull_all_gather(kind, world, dname):
    n_excluded = run_all_gather_case(kind, world, DTYPES[dname])
    if kind == "vitl_block" and world in (2, 8, 16):  # qkv (3072 rows) and fc1 (4096 rows) split into whole rows
        assert n_excluded > 0, "the exclusion branch never ran"


L2_HINT_CASES = [("synthetic", 3, torch.bfloat16), ("vitl_block", 5, torch.float32), ("vit10b_root", 8, torch.bfloat16),
                 ("vitl_block", 16, torch.bfloat16)]


def _no_l2_hint_main():
    assert os.environ.get("B200_COMM_L2_HINT") == "0"
    torch.cuda.set_device(0)
    for kind, world, dtype in L2_HINT_CASES:
        run_all_gather_case(kind, world, dtype)
        print(f"ok {kind} W={world} {dtype}")


@pytest.mark.gpu
def test_pull_all_gather_without_l2_hint():
    """The plain streaming loads and stores (l2_hint = 0).  B200_COMM_L2_HINT is read once per process, so this runs
    in a subprocess."""
    env = dict(os.environ)
    env["B200_COMM_L2_HINT"] = "0"
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "no_l2_hint"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert p.stdout.count("ok ") == len(L2_HINT_CASES), p.stdout


# ------------------------------------------------------------------------------------------------
# all-gather fused into the GEMM
# ------------------------------------------------------------------------------------------------
def gemm_unit_specs(name, N, K):
    """The weight between its LayerNorm and its bias, as in a block: the group does not start the buffer."""
    norm = "norm1" if name == "attn.qkv.weight" else "norm2"
    return [(f"{norm}.weight", (K,)), (f"{norm}.bias", (K,)), (name, (N, K)), (name.replace("weight", "bias"), (N,))]


# id: (W, weight name, N, K, M, block_n, cluster, max_ctas, epilogue).  Rows per slab: 1920 (a multiple of 128 but not
# of 256), 480, 200, 96 and 72 (less than a tile: one tile waits for several slabs); slab bytes are whole 16 KiB chunks
# only for the ViT-10B qkv and N = 480; every N but 15360 and 1152 / 128 leaves an N tail; max_ctas = 1 leaves all the
# pulling to one copier warp (and forces cluster 1).
GEMM_CASES = {
    "vit10b_qkv_w8": (8, "attn.qkv.weight", 15360, 5120, 264, 256, 1, 0, "bias"),
    "vit10b_qkv_w8_pairs": (8, "attn.qkv.weight", 15360, 5120, 264, 128, 2, 0, "bias_residual"),
    "vit10b_qkv_w8_one_cta": (8, "attn.qkv.weight", 15360, 5120, 136, 256, 1, 1, "gelu_preact"),
    "n960_k320_w2": (2, "mlp.fc1.weight", 960, 320, 200, 256, 1, 0, "gelu_preact"),
    "n960_k320_w2_pairs": (2, "mlp.fc1.weight", 960, 320, 200, 128, 2, 2, "bias_residual"),
    "n960_k320_w2_one_cta": (2, "mlp.fc1.weight", 960, 320, 77, 128, 1, 1, "bias"),
    "n600_k256_w3_pairs": (3, "mlp.fc1.weight", 600, 256, 129, 128, 2, 0, "gelu_preact"),
    "n480_k512_w5_pairs": (5, "attn.qkv.weight", 480, 512, 300, 256, 2, 4, "bias_residual"),
    "n1152_k328_w16": (16, "mlp.fc1.weight", 1152, 328, 256, 256, 1, 0, "gelu_preact"),
    "n1152_k328_w16_pairs": (16, "mlp.fc1.weight", 1152, 328, 256, 128, 2, 2, "bias_residual"),
    "n1152_k328_w16_one_cta": (16, "mlp.fc1.weight", 1152, 328, 100, 256, 1, 1, "bias"),
}
AG_CHUNK = 16384  # bytes per pull of the copier warp (kAgChunkBytes)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GEMM_CASES))
def test_all_gather_fused_into_gemm(case):
    """y = epilogue(x w^T) while the GEMM's copier warps pull w's row slabs from the virtual peers.  Five back-to-back
    launches per rank reuse the same counters.  After each: the gathered rows are w_full bit for bit and the rest of the
    unit buffer is untouched, every slab counter is complete, and y (and the pre-activation) is bitwise the same GEMM
    run on w_full without the gather (tile order does not change any tile's arithmetic) and close to float64."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    world, name, N, K, M, block_n, cluster, max_ctas, epi = GEMM_CASES[case]
    lay = UnitLayout.build("blocks.0", gemm_unit_specs(name, N, K), world, False)
    g = next(x for x in lay.groups if x.name == name)
    gen = torch.Generator(device="cuda").manual_seed(seed_of(N, K, world))
    shards = [(torch.randn(lay.shard_numel, generator=gen, device="cuda") * 0.05).to(torch.bfloat16)
              for _ in range(world)]
    full_ref = lay.full_from_shards(shards, sentinel(lay.full_numel, torch.bfloat16))
    w_full = lay.param_views(full_ref)[name].contiguous()
    x = torch.randn(M, K, generator=gen, device="cuda").to(torch.bfloat16)
    bias = torch.randn(N, generator=gen, device="cuda").to(torch.bfloat16)
    res = torch.randn(M, N, generator=gen, device="cuda").to(torch.bfloat16) if epi == "bias_residual" else None
    gelu = epi == "gelu_preact"

    def gemm(w, ag=()):
        y = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        pre = torch.empty(M, N, dtype=torch.bfloat16, device="cuda") if gelu else None
        co.gemm_raw(x, K, 0, w, K, 0, y, N, M, N, K, bias=bias, residual=res, ld_res=N if res is not None else 0,
                    aux_out=pre, ld_aux_out=N if gelu else 0, act=co.ACT_GELU if gelu else co.ACT_NONE,
                    block_n=block_n, cluster=cluster, max_ctas=max_ctas, ag=ag)
        return y, pre

    y_ref, pre_ref = gemm(w_full)
    pre64 = x.double() @ w_full.double().t() + bias.double()
    y64 = gelu_ref(pre64) if gelu else pre64 + (res.double() if res is not None else 0)
    assert_close_elementwise(y_ref, y64, what=f"{case}: y without the gather vs float64")
    chunks_per_slab = -(-g.shard_len * 2 // AG_CHUNK)
    lo, hi = g.full_offset, g.full_offset + world * g.shard_len
    for rank in ranks(world):
        be = virtual_backend(world, rank)
        assert name in Sm100Backend.fusable_params(be, lay)
        full = torch.empty(lay.full_numel, dtype=torch.bfloat16, device="cuda")
        be._peer[shards[rank].data_ptr()] = [s.data_ptr() for s in shards]
        spec = Sm100Backend.ag_fuse_spec(be, lay, shards[rank], full, name)
        assert spec[:4] == [world, rank, N // world, g.shard_len * 2]
        flags = be._seg_cache[("flags", full.data_ptr(), name)]
        w_view = lay.param_views(full)[name]
        for it in range(5):
            full.copy_(sentinel(lay.full_numel, torch.bfloat16))
            y, pre = gemm(w_view, spec)
            torch.cuda.synchronize()
            where = f"{case} rank {rank} launch {it}"
            assert_bitwise(f"{where}: gathered weight", full[lo:hi], full_ref[lo:hi])
            assert_bitwise(f"{where}: unit buffer outside the weight", torch.cat([full[:lo], full[hi:]]),
                           sentinel(lay.full_numel - (hi - lo), torch.bfloat16))
            cnt = flags[:world + 1].tolist()
            assert cnt[:world] == [chunks_per_slab] * world, f"{where}: slab counters {cnt[:world]}"
            assert cnt[world] >= world * chunks_per_slab + 1, f"{where}: chunk counter {cnt[world]}"
            if max_ctas == 1:
                assert cnt[world] == world * chunks_per_slab + 1, f"{where}: one copier warp, counter {cnt[world]}"
            assert_bitwise(f"{where}: y vs the GEMM without the gather", y, y_ref)
            if gelu:
                assert_bitwise(f"{where}: pre-activation vs the GEMM without the gather", pre, pre_ref)
    if gelu:
        assert_close_elementwise(pre_ref, pre64, what=f"{case}: pre-activation vs float64")


# ------------------------------------------------------------------------------------------------
# CPU meta-tests
# ------------------------------------------------------------------------------------------------
def _cpu_peers(world, n, seed, dtype=torch.float32):
    return [grad_values(n, seed_of(seed, r), dtype, device="cpu") for r in range(world)]


def test_replay_is_the_ordered_fp32_sum_on_normal_values():
    """Away from subnormals the replay is the plain left-to-right fp32 sum from +0.0 in the staggered order, times
    float32(1 / W)."""
    for world in WORLDS:
        for rank in ranks(world):
            sl = [s.to(torch.bfloat16) for s in _cpu_peers(world, 4099, world)]
            sl = [torch.where(s.float().abs() < FLT_MIN, torch.zeros_like(s), s) for s in sl]
            acc = np.zeros(4099, dtype=np.float32)
            for k in range(world):
                acc = acc + sl[(rank + k) % world].float().numpy()
            ref = acc * np.float32(1.0 / world)
            got = rs_replay(sl, rank).numpy()
            assert np.array_equal(got.view(np.int32), ref.view(np.int32)), (world, rank)


def test_replay_flushes_subnormals_and_starts_from_positive_zero():
    sl = [torch.tensor([-0.0, 3e-39, -3e-39, 2.0 ** -120], dtype=torch.float32) for _ in range(2)]
    got = rs_replay(sl, 0)
    assert got.tolist() == [0.0, 0.0, 0.0, 2.0 ** -120]
    assert not bool(torch.signbit(got[:3]).any()), "+0.0 plus -0 (or a flushed negative subnormal) is +0"


def test_reduce_scatter_checker_rejects_mutants():
    """Peers summed in reverse order, the 1 / W scale missing, one peer dropped, one segment shifted by a vector."""
    world, rank = 5, 3
    lay = unit_layout("synthetic", world)
    peers = _cpu_peers(world, lay.full_numel, 7, torch.bfloat16)
    sl = shard_slices(lay, peers, rank)
    good = rs_replay(sl, rank)
    check_reduce_scatter(sl, rank, good)
    reverse = [(rank - k) % world for k in range(world)]
    dropped = [(rank + k) % world for k in range(world - 1)]
    g = next(x for x in lay.groups if x.name == "mlp.fc1.weight")
    shifted = good.clone()
    shifted[g.shard_offset + 8: g.shard_offset + g.shard_len] = good[g.shard_offset: g.shard_offset + g.shard_len - 8]
    mutants = {"reverse order": rs_replay(sl, rank, order=reverse), "no 1 / W": rs_replay(sl, rank, scale=1.0),
               "peer dropped": rs_replay(sl, rank, order=dropped), "segment shifted": shifted}
    for what, bad in mutants.items():
        with pytest.raises(AssertionError, match="fp32 replay"):
            check_reduce_scatter(sl, rank, bad)
    # the float64 bound alone also rejects the arithmetic mutants
    s64 = sum(s.double() for s in sl)
    a64 = sum(s.double().abs() for s in sl)
    for what in ("no 1 / W", "peer dropped"):
        with pytest.raises(AssertionError):
            assert_within(what, mutants[what], s64 / world, (world + 1.01) * U * a64 / world + (world + 2) * FLT_MIN)


def test_sumsq_checker_rejects_a_missing_start_value():
    out = torch.linspace(-0.1, 0.1, 10000)
    ref = out.double().square().sum()
    check_sumsq((0.75 + ref).float(), 0.75, out, 5, 3, 8)
    with pytest.raises(AssertionError, match="sumsq"):
        check_sumsq(ref.float(), 0.75, out, 5, 3, 8)


def _adamw_f32(w0, m0, v0, g, hp, step, bc_fp32, ieee_rcp=True):
    """The fp32 AdamW step the kernels run.  bc_fp32=True is the mutant: 1 - beta^t formed with an fp32 powf."""
    f = np.float32
    lr, b1, b2, eps, wd = (f(t) for t in hp)
    if bc_fp32:
        bc1, bc2 = f(1) - np.power(b1, f(step)), f(1) - np.power(b2, f(step))
    else:
        bc1, bc2 = f(1.0 - float(b1) ** step), f(1.0 - float(b2) ** step)
    inv1, inv2 = f(1) / bc1, f(1) / bc2
    if not ieee_rcp:  # the device's approximate reciprocal: one ulp off
        inv1, inv2 = np.nextafter(inv1, f(0)), np.nextafter(inv2, f(np.inf))
    # fp32 scalars as Python floats (exact): torch then rounds every product and sum to fp32
    lr, b1, b2, eps, inv1, inv2, c1, c2, decay = (float(t) for t in (lr, b1, b2, eps, inv1, inv2, f(1) - b1,
                                                                     f(1) - b2, f(1) - lr * wd))
    m = b1 * m0 + c1 * g
    v = b2 * v0 + c2 * g * g
    w = w0 * decay - lr * (m * inv1) / (torch.sqrt(v * inv2) + eps)
    return w, m, v


def test_adamw_checkers_reject_the_fp32_bias_correction():
    """At step 2 an fp32 powf leaves 1 - beta2^2 several ulps off, a few 1e-6 of every update: both the float64
    AdamW checker and the comparison with adamw_split reject it, while an IEEE against an approximate reciprocal of the
    correct bias correction passes."""
    hp = (_f32(1e-3), _f32(0.9), _f32(0.999), _f32(1e-8), _f32(0.1))
    gen = torch.Generator().manual_seed(0)
    n = 4096
    w0 = torch.randn(n, generator=gen) * 0.02
    w0[::4] = torch.randn(n // 4, generator=gen) * 1e-5
    m0 = torch.randn(n, generator=gen) * 1e-3
    v0 = (torch.randn(n, generator=gen) * 1e-3).square()
    g = grad_values(n, 5, torch.float32, device="cpu")
    for step in (2, 3):
        split = _adamw_f32(w0, m0, v0, g, hp, step, bc_fp32=False, ieee_rcp=False)
        good = _adamw_f32(w0, m0, v0, g, hp, step, bc_fp32=False)
        bad = _adamw_f32(w0, m0, v0, g, hp, step, bc_fp32=True)
        check_adamw(w0, m0, v0, g, 1.0, hp, step, *good)
        check_fused_matches_split(m0, v0, g, hp, step, good, split)
        with pytest.raises(AssertionError, match="adamw w"):
            check_adamw(w0, m0, v0, g, 1.0, hp, step, *bad)
        with pytest.raises(AssertionError, match="fused AdamW w"):
            check_fused_matches_split(m0, v0, g, hp, step, bad, split)


def test_all_gather_checker_rejects_bytes_in_an_excluded_group():
    world = 2
    lay = unit_layout("vitl_block", world)
    be = virtual_backend(world, 0, device="cpu", C=_fake_C())
    exclude = Sm100Backend.fusable_params(be, lay)
    assert set(exclude) == {"attn.qkv.weight", "mlp.fc1.weight"}
    shards = [random_bits(lay.shard_numel, torch.bfloat16, r, device="cpu") for r in range(world)]
    full_ref = lay.full_from_shards(shards, torch.empty(lay.full_numel, dtype=torch.bfloat16))
    out = full_ref.clone()
    check_all_gather(lay, full_ref, out, ())
    with pytest.raises(AssertionError, match="exclude"):
        check_all_gather(lay, full_ref, out, exclude)
    g = next(x for x in lay.groups if x.name == "mlp.fc1.weight")
    for x in lay.groups:
        if x.name in exclude:
            out[x.full_offset: x.full_offset + world * x.shard_len] = sentinel(world * x.shard_len, out.dtype, "cpu")
    check_all_gather(lay, full_ref, out, exclude)
    out[g.full_offset + 5] = full_ref[g.full_offset + 5]  # one stray element
    with pytest.raises(AssertionError, match="exclude"):
        check_all_gather(lay, full_ref, out, exclude)


def _fake_C():
    return types.SimpleNamespace(ag_chunk_bytes=lambda: AG_CHUNK, rs_chunk_vecs=lambda: 512)


@pytest.mark.parametrize("world", range(2, 17))
def test_ag_fuse_spec_allocates_a_counter_per_slab_and_the_chunk_counter(world):
    """The GEMM zeroes world + 1 words at spec[5] and counts pulled chunks in flags[world]: the tensor behind that
    pointer must hold at least world + 1 int32 counters for every world size the extension accepts (up to 16)."""
    lay = UnitLayout.build("blocks.0", gemm_unit_specs("mlp.fc1.weight", 8 * world, 64), world, False)
    be = virtual_backend(world, world - 1, device="cpu", C=_fake_C())
    shard = torch.zeros(lay.shard_numel, dtype=torch.bfloat16)
    full = torch.zeros(lay.full_numel, dtype=torch.bfloat16)
    be._peer[shard.data_ptr()] = [(r + 1) << 40 for r in range(world)]
    spec = Sm100Backend.ag_fuse_spec(be, lay, shard, full, "mlp.fc1.weight")
    flags = be._seg_cache[("flags", full.data_ptr(), "mlp.fc1.weight")]
    assert len(spec) == 6 + world and spec[5] == flags.data_ptr()
    assert flags.dtype == torch.int32 and flags.is_contiguous()
    assert flags.numel() >= world + 1, (f"ag_fuse_spec allocated {flags.numel()} counters at W = {world}; the GEMM "
                                        f"zeroes and uses world + 1 = {world + 1} (flags[world] is the chunk counter)")
    assert Sm100Backend.ag_fuse_spec(be, lay, shard, full, "mlp.fc1.weight")[5] == spec[5], "one set per weight"


if __name__ == "__main__":
    if sys.argv[1] == "no_l2_hint":
        _no_l2_hint_main()
