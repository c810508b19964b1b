"""Shared helpers for the CPU test-suite."""
import hashlib
import os
import re
import socket
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from vit_10b_fsdp_example_b200.config import ViTConfig  # noqa: E402

TINY = dict(image_size=32, patch_size=8, embed_dim=64, num_heads=4, num_blocks=3, mlp_ratio=2.0, num_classes=10)


def tiny_cfg(**kw):
    d = dict(TINY)
    d.update(kw)
    return ViTConfig(**d)


def sass_symbol_key(name):
    """A kernel symbol without its anonymous-namespace tag: nvcc derives `_GLOBAL__N__<hash>_<len><file>_<hash>` from
    the source file's path, so the same kernel has another mangled name in every checkout."""
    return re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+)(\w*?)_[0-9a-f]{8}", r"_GLOBAL__N__\1\2", name)


def sass_hash(obj, name):
    """SHA-256 of kernel `name`'s SASS in object `obj` (cuobjdump), instructions only, without their addresses."""
    out = subprocess.run(["cuobjdump", "-sass", "-fun", name, obj], capture_output=True, text=True, check=True).stdout
    ins = [re.sub(r"/\*[0-9a-f]{4,}\*/", "", ln).strip() for ln in out.splitlines() if ";" in ln]
    return hashlib.sha256("\n".join(ins).encode()).hexdigest()


def ptxas_usage(log):
    """{symbol key: [registers, spill store bytes, spill load bytes]} from `-Xptxas -v` output."""
    lines = log.splitlines()
    usage = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln:
            spill = next(x for x in lines[i + 1:] if "spill stores" in x)
            regs = next(x for x in lines[i + 1:] if re.search(r"Used \d+ registers", x))
            st, ld = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", spill).groups()
            usage[sass_symbol_key(ln.split("'")[1])] = [int(re.search(r"Used (\d+) registers", regs).group(1)), int(st),
                                                        int(ld)]
    return usage


def free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def autograd_vit_loss(cfg, params, images, target):
    """Plain PyTorch (autograd) ViT with timm semantics -- the oracle for the hand-written backward.

    params: dict name -> tensor (requires_grad) with names '<blocks.i.>norm1.weight', 'pos_embed' ...
    """
    B = images.shape[0]
    N, D, H, hd = cfg.num_patches, cfg.embed_dim, cfg.num_heads, cfg.head_dim
    P = cfg.patch_size
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, P, P)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=P).flatten(2).transpose(1, 2)
    x = x + params["pos_embed"].view(1, N, D)
    for i in range(cfg.num_blocks):
        g = lambda n: params[f"blocks.{i}.{n}"]  # noqa: E731
        h = F.layer_norm(x, (D,), g("norm1.weight"), g("norm1.bias"), 1e-5)
        qkv = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        att = ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1)
        a = (att @ v).transpose(1, 2).reshape(B, N, D)
        x = x + F.linear(a, g("attn.proj.weight"), g("attn.proj.bias"))
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        h = F.linear(F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))), g("mlp.fc2.weight"), g("mlp.fc2.bias"))
        x = x + h
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x.mean(dim=1), params["head.weight"], params["head.bias"])
    return F.cross_entropy(logits, target), logits


def full_params_of(model):
    """name -> fp32 tensor of the full (unsharded) parameters of a world-size-1 model."""
    out = {}
    for u in model.all_units:
        full = model.master_fp32(u)
        prefix = "" if u.name == "root" else u.name + "."
        for n, v in u.layout.param_views(full).items():
            out[prefix + n] = v.clone()
    return out


def full_grads_of(model):
    out = {}
    for u in model.all_units:
        prefix = "" if u.name == "root" else u.name + "."
        for n, v in u.layout.param_views(u.full_grad.float()).items():
            out[prefix + n] = v.clone()
    return out


def assert_close_elementwise(got, ref, rtol=2e-2, atol_rel=2e-2, what=""):
    """Per-element bound |got - ref| <= atol + rtol * |ref| with atol = atol_rel * mean|ref|.

    A max-normalised check (max|err| / max|ref|) is blind to errors in small-magnitude outputs; this one holds every
    element to a relative tolerance plus an absolute floor tied to the *typical* magnitude of the tensor (bf16 has
    2^-8 relative precision; sums of many bf16 products carry an absolute error proportional to the typical term)."""
    got, ref = got.float(), ref.float()
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    atol = atol_rel * ref.abs().mean().item() + 1e-12
    err = (got - ref).abs()
    bound = atol + rtol * ref.abs()
    bad = err > bound
    if bad.any():
        i = (err - bound).argmax().item()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of tolerance; worst: got "
                             f"{got.flatten()[i].item():.6g} ref {ref.flatten()[i].item():.6g} "
                             f"(atol {atol:.3g}, rtol {rtol})")
