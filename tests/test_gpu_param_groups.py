"""Optimizer parameter groups on the H100: the grouped AdamW kernels against float64 and bitwise against the plain
ones, the grouped AdamW fused into the reduce-scatter, the bf16 engine against torch.optim.AdamW with MAE-style groups,
CUDA-graph replay, the unchanged path without the flags, and the sm_90a build of the new kernels."""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from helpers import sass_hash, sass_symbol_key  # noqa: E402
from test_gpu_memory_bound_fp64 import _f32, adamw_state, check_adamw, check_split  # noqa: E402

U = 2.0 ** -24
HP = (1e-3, 0.9, 0.999, 1e-8, 0.1)  # lr, beta1, beta2, eps, wd
# three groups: (lr_scale, wd) = a decayed block, a no-decay group and a strongly scaled decayed stem
TABLE = [[1.0, 0.1], [0.75, 0.0], [0.0563, 0.1]]


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def alternating_groups(n, G=3):
    """Chunk c is in group c % G, except every 7th chunk, which is in group 0: neighbours always differ somewhere."""
    c = torch.arange(n // 64, device="cuda") % G
    c[::7] = 0
    return c.to(torch.uint8)


def per_element(lr, groups, table):
    """(lr * lr_scale in fp32, wd) of every element, as float64 tensors."""
    t = torch.tensor(table, dtype=torch.float32, device="cuda")
    idx = groups.long().repeat_interleave(64)
    lr_e = t[idx, 0] * torch.tensor(_f32(lr), dtype=torch.float32, device="cuda")
    return lr_e.double(), t[idx, 1].double()


def _merge(hi, lo):
    w = torch.empty(hi.numel(), dtype=torch.float32, device=hi.device)
    _co().merge_fp32(hi, lo, w)
    return w


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _bits_equal(a, b):
    return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------
# the grouped kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("flavour", ["split", "split_hyper", "fp32"])
def test_grouped_kernels_against_fp64(flavour, gdtype, ema):
    """Each element is updated by the fp64 AdamW step at its own group's lr * lr_scale and wd; the EMA operand changes
    nothing else (bitwise against the same grouped launch without it) and follows ema = d ema + (1 - d) w."""
    co = _co()
    lr, b1, b2, eps, wd = (_f32(t) for t in HP)
    table = torch.tensor(TABLE, dtype=torch.float32, device="cuda")
    coef = _f32(0.37)
    clip_t = torch.tensor([coef], device="cuda")
    for n in (8192, 64 * 131):
        groups = alternating_groups(n)
        lr_e, wd_e = per_element(lr, groups, TABLE)
        for step in (1, 10, 1000):
            w0, m0, v0 = adamw_state(n, step, seed=n + step)
            gen = torch.Generator(device="cuda").manual_seed(n * step)
            g = torch.randn(n, generator=gen, device="cuda").to(gdtype)
            g[::5] = 0
            m, v = m0.clone(), v0.clone()
            e0 = (w0 * 0.5).contiguous()
            if flavour == "fp32":
                w = w0.clone()
                ema_t = e0.clone() if ema else None
                co.adamw_fp32(w, m, v, g, clip_t, lr, b1, b2, eps, 123.0, step, ema=ema_t, ema_decay=0.9,
                              groups=groups, group_hyper=table)
                if ema:
                    w2, m2, v2 = w0.clone(), m0.clone(), v0.clone()
                    co.adamw_fp32(w2, m2, v2, g, clip_t, lr, b1, b2, eps, 123.0, step, groups=groups,
                                  group_hyper=table)
                    assert _bits_equal(w, w2) and _bits_equal(m, m2) and _bits_equal(v, v2)
                    ema_new = ema_t
            else:
                hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
                lo = torch.empty(n, dtype=torch.int16, device="cuda")
                co.split_fp32(w0, hi, lo)
                ehi, elo = torch.empty_like(hi), torch.empty_like(lo)
                co.split_fp32(e0, ehi, elo)
                state = [hi.clone(), lo.clone(), m0.clone(), v0.clone()]
                if flavour == "split":  # the host wd is ignored: the table carries it
                    args = (clip_t, lr, b1, b2, eps, 123.0, step)
                    kw = {}
                else:  # the device block [lr, step] overrides the host lr / step
                    args = (clip_t, 10 * lr, b1, b2, eps, 123.0, step + 7)
                    kw = {"hyper": torch.tensor([lr, float(step)], device="cuda")}
                co.adamw_split(hi, lo, m, v, g, *args, **kw, ema=(ehi, elo) if ema else None, ema_decay=0.9,
                               groups=groups, group_hyper=table)
                w = _merge(hi, lo)
                check_split(hi, lo, w)
                if ema:
                    co.adamw_split(*state, g, *args, **kw, groups=groups, group_hyper=table)
                    for a, b in zip((hi, lo, m, v), state):
                        assert _bits_equal(a, b)
                    ema_new = _merge(ehi, elo)
            check_adamw(w0, m0, v0, g, coef, (lr_e, b1, b2, eps, wd_e), step, w, m, v)
            if ema:
                d, k = _f32(0.9), _f32(1.0 - _f32(0.9))
                e64 = d * e0.double() + k * w.double()
                assert bool(((ema_new.double() - e64).abs() <= 2 * U * ((k * w.double()).abs() + e64.abs())).all())


@pytest.mark.gpu
@pytest.mark.parametrize("flavour", ["split", "split_hyper", "fp32"])
def test_zero_gradient_leaves_no_decay_chunks_bitwise_and_decays_the_rest(flavour):
    """g = 0 and zero moments: the Adam term is exactly 0, so a no-decay chunk keeps its bits and a decayed one becomes
    w * decay with decay = fp32(1 - fp32(lr * s) wd) (the product lr * s * wd rounded once by an fma, or twice)."""
    co = _co()
    n = 64 * 97
    lr, wd = _f32(1e-3), _f32(0.1)
    groups = alternating_groups(n)
    table = torch.tensor(TABLE, dtype=torch.float32, device="cuda")
    w0, _, _ = adamw_state(n, 1, seed=11)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    g = torch.zeros(n, device="cuda")
    if flavour == "fp32":
        w = w0.clone()
        co.adamw_fp32(w, m, v, g, None, lr, 0.9, 0.999, 1e-8, wd, 1, groups=groups, group_hyper=table)
    else:
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        lo = torch.empty(n, dtype=torch.int16, device="cuda")
        co.split_fp32(w0, hi, lo)
        hyper = torch.tensor([lr, 1.0], device="cuda") if flavour == "split_hyper" else None
        co.adamw_split(hi, lo, m, v, g, None, lr, 0.9, 0.999, 1e-8, wd, 1, hyper, groups=groups, group_hyper=table)
        w = _merge(hi, lo)
    idx = groups.long().repeat_interleave(64).cpu().numpy()
    wn, w0n = w.cpu().numpy(), w0.cpu().numpy()
    f = np.float32
    ok = np.zeros(n, dtype=bool)
    for gi, (s, gwd) in enumerate(TABLE):
        sel = idx == gi
        if gwd == 0.0:
            assert np.array_equal(wn[sel].view(np.int32), w0n[sel].view(np.int32)), gi
            ok |= sel
            continue
        lr_s = f(f(lr) * f(s))
        fused = f(1.0 - float(lr_s) * float(f(gwd)))       # fma: one rounding
        split = f(f(1.0) - f(lr_s * f(gwd)))                 # product rounded first
        for decay in (fused, split):
            ok |= sel & (wn.view(np.int32) == (w0n * decay).astype(np.float32).view(np.int32))
    assert ok.all(), f"{int((~ok).sum())} elements differ"


@pytest.mark.gpu
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("flavour", ["split", "split_hyper", "fp32"])
def test_one_group_of_scale_one_reproduces_the_plain_kernel_bitwise(flavour, gdtype, ema):
    co = _co()
    n = 64 * 203
    lr, b1, b2, eps, wd = (_f32(t) for t in HP)
    groups = torch.zeros(n // 64, dtype=torch.uint8, device="cuda")
    table = torch.tensor([[1.0, wd]], dtype=torch.float32, device="cuda")
    clip_t = torch.tensor([_f32(0.6)], device="cuda")
    for step in (1, 3, 500):
        w0, m0, v0 = adamw_state(n, step, seed=step)
        g = (torch.randn(n, device="cuda") * 1e-2).to(gdtype)
        runs = []
        for grouped in (False, True):
            grp = {"groups": groups, "group_hyper": table} if grouped else {}
            m, v = m0.clone(), v0.clone()
            if flavour == "fp32":
                w = w0.clone()
                e = (w0 * 0.3).contiguous() if ema else None
                co.adamw_fp32(w, m, v, g, clip_t, lr, b1, b2, eps, wd, step, ema=e, ema_decay=0.99, **grp)
                runs.append([w, m, v] + ([e] if ema else []))
            else:
                hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
                lo = torch.empty(n, dtype=torch.int16, device="cuda")
                co.split_fp32(w0, hi, lo)
                e = (hi.clone(), lo.clone()) if ema else None
                hyper = torch.tensor([lr, float(step)], device="cuda") if flavour == "split_hyper" else None
                co.adamw_split(hi, lo, m, v, g, clip_t, lr, b1, b2, eps, wd, step, hyper, ema=e, ema_decay=0.99, **grp)
                runs.append([hi, lo, m, v] + (list(e) if ema else []))
        for a, b in zip(*runs):
            assert _bits_equal(a, b), step


@pytest.mark.gpu
def test_bad_group_arguments_are_refused():
    co = _co()
    n = 256
    hi = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    lo = torch.zeros(n, dtype=torch.int16, device="cuda")
    m, v, g = (torch.zeros(n, device="cuda") for _ in range(3))
    table = torch.tensor([[1.0, 0.1]], device="cuda")
    ok = torch.zeros(n // 64, dtype=torch.uint8, device="cuda")
    for groups, gh, what in [(ok[:-1], table, "chunk groups"), (ok.int(), table, "uint8"),
                             (ok, table.double(), "uint8"), (ok.cpu(), table, "device"),
                             (ok, table.view(2, 1), r"\[G, 2\]")]:
        with pytest.raises(RuntimeError, match=what):
            co.adamw_split(hi, lo, m, v, g, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, groups=groups, group_hyper=gh)
    with pytest.raises(RuntimeError, match="n % 64 == 0"):
        co.adamw_fp32(m[:100], v[:100], g[:100].clone(), g[:100], None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1,
                      groups=ok[:1], group_hyper=table)


# ------------------------------------------------------------------------------------------------
# the grouped AdamW fused into the reduce-scatter (one GPU, virtual peers)
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("step", [1, 10, 1000])
def test_grouped_adamw_fused_into_reduce_scatter(step):
    """The real group tables of a ViT-L block (flat and per-parameter) and of the ViT-10B root unit, through the
    reduce-scatter kernel: against the fp64 step at each element's group, and against the grouped adamw_split run on
    the same state with the unfused reduce-scatter's gradient."""
    from test_gpu_comm_kernels import (VIT10B, VITL, check_fused_matches_split, grad_values, rs_replay, run_reduce_scatter,
                                       seed_of, sentinel, shard_slices, unit_layout, virtual_backend)

    from vit_10b_fsdp_example_b200.parallel import param_groups as pg

    co = _co()
    hyper = [1e-3, 0.9, 0.999, 1e-8, 0.1, float(step)]
    lr, b1, b2, eps, wd = (_f32(t) for t in hyper[:5])
    for kind, world, rank, max_ctas in [("vitl_block", 8, 7, 0), ("vitl_block_flat", 4, 1, 3), ("vit10b_root", 8, 0, 132)]:
        lay = unit_layout(kind, world)
        cfg = VIT10B if kind == "vit10b_root" else VITL
        ug = pg.build_unit_groups(cfg, lay, rank, wd, 0.75, "cuda")
        n = lay.shard_numel
        peers = [grad_values(lay.full_numel, seed_of(step, world, r), torch.bfloat16) for r in range(world)]
        be = virtual_backend(world, rank)
        gmean = rs_replay(shard_slices(lay, peers, rank), rank)
        w0, m0, v0 = adamw_state(n, step, seed=seed_of(step, world, 3))
        hi = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        lo = torch.empty(n, dtype=torch.int16, device="cuda")
        co.split_fp32(w0, hi, lo)
        m, v = m0.clone(), v0.clone()
        out = sentinel(n, torch.float32)
        run_reduce_scatter(be, lay, peers, out, None, max_ctas,
                           adam=(hi, lo, m, v, hyper, ug.chunk_groups, ug.group_hyper))
        w = _merge(hi, lo)
        torch.cuda.synchronize()
        check_split(hi, lo, w)
        rows = ug.group_hyper.cpu().tolist()
        lr_e, wd_e = per_element(lr, ug.chunk_groups, rows)
        check_adamw(w0, m0, v0, gmean, 1.0, (lr_e, b1, b2, eps, wd_e), step, w, m, v)
        hi2, lo2 = torch.empty_like(hi), torch.empty_like(lo)
        co.split_fp32(w0, hi2, lo2)
        m2, v2 = m0.clone(), v0.clone()
        co.adamw_split(hi2, lo2, m2, v2, gmean, None, lr, b1, b2, eps, wd, step, groups=ug.chunk_groups,
                       group_hyper=ug.group_hyper)
        check_fused_matches_split(m0, v0, gmean, (lr_e, b1, b2, eps, wd_e), step, (w, m, v), (_merge(hi2, lo2), m2, v2))


# ------------------------------------------------------------------------------------------------
# the bf16 engine on one GPU
# ------------------------------------------------------------------------------------------------
def _cfg():
    from vit_10b_fsdp_example_b200.config import ViTConfig

    return ViTConfig(image_size=112, patch_size=14, embed_dim=320, num_heads=2, num_blocks=3, mlp_ratio=4.0,
                     num_classes=96, class_token=True, reg_tokens=2, init_values=1e-2, qk_norm=True)


def _data(n=3, B=8):
    g = torch.Generator().manual_seed(0)
    return [(torch.randn(B, 3, 112, 112, generator=g).cuda(), torch.randint(0, 96, (B,), generator=g).cuda())
            for _ in range(n)]


def _model(**kw):
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    model = FSDPViT(_cfg(), device=torch.device("cuda"), dtype=torch.bfloat16, seed=4)
    return model, ShardedAdamW(model, lr=2e-3, weight_decay=0.1, **kw)


def _unit_views(unit, flat):
    """timm name -> view of a world-1 unit's shard-shaped buffer (the shard layout is the full layout at W = 1)."""
    prefix = "" if unit.name == "root" else unit.name + "."
    return {prefix + k: t for k, t in unit.layout.param_views(flat).items()}


@pytest.mark.gpu
def test_engine_update_matches_torch_adamw_with_mae_groups():
    """Three bf16 steps with --layer_decay 0.75: after each backward the engine's reduced fp32 gradient (times the clip
    coefficient) is handed to torch.optim.AdamW with one group per (layer, decay) pair on an fp32 copy of the master,
    lr = base * 0.75 ** (L + 1 - layer) and weight_decay 0 for the no-decay set; the engine's new master must match it
    to fp32 rounding."""
    from test_param_groups import expected_layer

    model, opt = _model(layer_decay=0.75)
    L, d = model.cfg.num_blocks, 0.75
    lrs = [2e-3, 1.4e-3, 7e-4]
    for (x, y), lr in zip(_data(), lrs):
        opt.param_groups[0]["lr"] = lr
        model.forward_backward(x, y)
        model.clip_grad_norm_(1.0)
        coef = float(model._clip_coef.item())
        params, groups = {}, {}
        for u in model.all_units:
            w = _unit_views(u, model.master_fp32(u))
            gr = _unit_views(u, u.shard_grad)
            for n, t in w.items():
                p = torch.nn.Parameter(t.clone())
                p.grad = gr[n].float() * coef  # fp32, as the kernel scales the (bf16 at W = 1) gradient
                no_decay = t.dim() <= 1 or n in ("pos_embed", "cls_token", "reg_token")
                key = (expected_layer(n, L), no_decay)
                groups.setdefault(key, {"params": [], "weight_decay": 0.0 if no_decay else 0.1,
                                        "lr": lr * d ** (L + 1 - key[0])})["params"].append(p)
                params[n] = p
        ref = torch.optim.AdamW(list(groups.values()), lr=lr)
        for u in model.all_units:  # the moments carried over from the previous step
            m_v = _unit_views(u, u.exp_avg), _unit_views(u, u.exp_avg_sq)
            for n in m_v[0]:
                ref.state[params[n]] = {"step": torch.tensor(float(opt.state[u.name]["step"])),
                                        "exp_avg": m_v[0][n].clone(), "exp_avg_sq": m_v[1][n].clone()}
        ref.step()
        opt.step()
        for u in model.all_units:
            got = _unit_views(u, model.master_fp32(u))
            for n, t in got.items():
                torch.testing.assert_close(t, params[n].detach(), rtol=2e-6, atol=2e-8, msg=n)


@pytest.mark.gpu
def test_cuda_graph_replay_matches_eager_bitwise():
    """The grouped optimizer step replayed from a CUDA graph (device lr / step, the tables recorded once) gives bitwise
    the masters and moments of eager steps from the same gradients, at four scheduled learning rates."""
    data = _data()
    a, opt_a = _model(layer_decay=0.75)
    b, opt_b = _model(layer_decay=0.75)
    a.forward_backward(*data[0])
    for ua, ub in zip(a.all_units, b.all_units):
        ub.shard_grad.copy_(ua.shard_grad)
    lrs = [2e-3, 1.5e-3, 1e-3, 5e-4]
    for lr in lrs:
        opt_a.param_groups[0]["lr"] = lr
        opt_a.step()
    opt_b.lr_on_device = True
    opt_b.param_groups[0]["lr"] = lrs[0]
    opt_b.push_lr()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt_b.step()
    for lr in lrs:
        opt_b.param_groups[0]["lr"] = lr
        opt_b.push_lr()
        graph.replay()
    torch.cuda.synchronize()
    for ua, ub in zip(a.all_units, b.all_units):
        for t in ("hi", "lo", "exp_avg", "exp_avg_sq"):
            assert _bits_equal(getattr(ua, t), getattr(ub, t)), (ua.name, t)
    # and a whole graphed training step trains with the groups
    from vit_10b_fsdp_example_b200.parallel import GraphedTrainStep

    model, opt = _model(layer_decay=0.75)
    step = GraphedTrainStep(model, opt, clip_grad_norm=1.0, warmup=2)
    losses = [step(*data[i % 3]).item() for i in range(5)]
    assert step.graph is not None and all(np.isfinite(losses))


@pytest.mark.gpu
def test_without_the_flags_the_update_is_the_plain_kernels_bitwise():
    """With both flags off ShardedAdamW launches exactly what it launched before parameter groups existed: the same
    adamw_split calls with the same arguments (replayed here by hand on a copy of the state)."""
    model, opt = _model()
    assert opt.groups is None
    x, y = _data(1)[0]
    model.forward_backward(x, y)
    model.clip_grad_norm_(1.0)
    coef = model._clip_coef.clone()
    before = [[t.clone() for t in (u.hi, u.lo, u.exp_avg, u.exp_avg_sq)] for u in model.all_units]
    opt.step()
    co = _co()
    hyper = torch.tensor([2e-3, 1.0], device="cuda")
    for u, st in zip(model.all_units, before):
        co.adamw_split(*st, u.shard_grad, coef, 2e-3, 0.9, 0.999, 1e-8, 0.1, 1, hyper)
        for a, b in zip((u.hi, u.lo, u.exp_avg, u.exp_avg_sq), st):
            assert _bits_equal(a, b), u.name


# ------------------------------------------------------------------------------------------------
# build: the new kernels compile for sm_90a without spills or calls; the existing ones are unchanged
# ------------------------------------------------------------------------------------------------
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
GROUPED_NAMES = ("adamw_split_grouped_kernel", "adamw_split_ema_grouped_kernel", "adamw_fp32_grouped_kernel",
                 "adamw_fp32_ema_grouped_kernel")


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("cuobjdump") is None, reason="needs nvcc and cuobjdump")
def test_grouped_kernels_compile_for_sm90a_and_the_comm_kernels_stay_light(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    found = {}
    for src in ("elementwise.cu", "comm.cu"):
        obj = str(tmp_path / f"{src}.o")
        res = subprocess.run([NVCC, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                              os.path.join(build_ext.CSRC, src), "-o", obj], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-2000:]
        lines = (res.stdout + res.stderr).splitlines()
        for i, ln in enumerate(lines):
            if "Compiling entry function" in ln:
                found[(src, ln.split("'")[1])] = next(x for x in lines[i + 1:] if "spill stores" in x)
        if src == "elementwise.cu":
            new = [n for s, n in found if s == src and any(k in n for k in GROUPED_NAMES)]
            assert len(new) == 8, new  # {split, split + EMA, fp32, fp32 + EMA} x {bf16, fp32 gradient}
            for name in new:
                assert "0 bytes spill stores, 0 bytes spill loads" in found[(src, name)], name
                sass = subprocess.run(["cuobjdump", "-sass", "-fun", name, obj], capture_output=True, text=True).stdout
                assert "EXIT" in sass and " CALL" not in sass, name
            golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_before_swiglu.json")))
            ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
            if ver == golden["nvcc"]:
                sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
                names = {sass_symbol_key(n): n for n in re.findall(r"Function : (\S+)", sass)}
                for key, h in golden["objects"]["elementwise.cu"].items():
                    assert sass_hash(obj, names[key]) == h, f"SASS of pre-existing kernel {key} changed"
        else:
            txt = subprocess.run(["cuobjdump", "-res-usage", obj], capture_output=True, text=True).stdout
            rows = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)", txt)
            rs = [r for r in rows if "reduce_scatter_kernel" in r[0]]
            assert len(rs) == 5
            for name, reg, shared in rows:
                assert int(reg) <= 96 and int(shared) == 0, (name, reg, shared)
            for (s, name), v in found.items():
                if s == src:
                    assert "0 bytes spill stores, 0 bytes spill loads" in v, name
