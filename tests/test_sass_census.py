"""The built sm_90a objects really contain what the design claims (cuobjdump -sass of the in-tree build, CPU only):
wgmma MMAs fed by TMA through mbarrier pipelines in every GEMM / attention instantiation, TMA stores in the GEMM, in-switch
multimem reductions and system-scope flags in the collectives, bulk-copy pipelines in the streaming LayerNorm backward
-- and no legacy mma.sync (HMMA) tensor-core code anywhere."""
import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vit_10b_fsdp_example_b200", "csrc", "build")
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sass_summary  # noqa: E402

pytestmark = pytest.mark.skipif(
    shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(BUILD, "gemm_sm90.cu.o")),
    reason="needs cuobjdump and the in-tree build (python -m vit_10b_fsdp_example_b200.build_ext)")


@pytest.fixture(scope="module")
def census():
    return sass_summary.census(BUILD)


def _has(counter, prefix):
    return any(op.startswith(prefix) for op in counter)


def test_every_gemm_instantiation_is_a_wgmma_tma_kernel(census):
    kernels = {k: c for k, c in census["gemm_sm90.cu.o"].items() if "gemm_bf16_sm90_kernel" in k}
    assert len(kernels) >= 8
    for name, c in kernels.items():
        assert _has(c, "HGMMA.64"), name              # wgmma.mma_async m64nNk16
        assert _has(c, "WARPGROUP.DEPBAR"), name      # wgmma.wait_group: MMAs stay in flight across k-blocks
        assert _has(c, "UTMALDG.4D"), name            # TMA tensor loads of both operands
        assert _has(c, "SYNCS.PHASECHK"), name        # mbarrier full / empty ring between producer and consumers
        assert _has(c, "UTMASTG"), name               # TMA store of the output tile
        assert _has(c, "LDG.E.NA.128"), name          # copier warp of the fused all-gather (peer loads)


@pytest.mark.parametrize("hd", [64, 128, 160])
@pytest.mark.parametrize("family", ["attn_fwd_sm90_kernel<{hd}>", "attn_bwd_sm90_kernel<{hd}, 0>",
                                    "attn_bwd_sm90_kernel<{hd}, 1>"])
def test_attention_kernels_use_wgmma_and_tma(census, family, hd):
    name = family.format(hd=hd)
    kernels = {k: c for k, c in census["attention_sm90.cu.o"].items() if k.endswith(name)}
    assert len(kernels) == 1, name
    for c in kernels.values():
        for prefix in ("HGMMA.64", "UTMALDG.4D", "SYNCS.PHASECHK"):
            assert _has(c, prefix), (name, prefix)


def test_collectives_reduce_in_the_switch_and_signal_at_system_scope(census):
    comm = census["comm.cu.o"]
    nvls = [c for k, c in comm.items() if k.endswith("reduce_scatter_kernel<true, true, false>")
            or k.endswith("reduce_scatter_kernel<true, true, true>") or k.endswith("all_reduce_kernel<true>")]
    assert len(nvls) == 3
    for c in nvls:
        assert _has(c, "LDGMC.E.F32ADD.BF16")         # multimem.ld_reduce.add.bf16x2: the reduction happens in NVSwitch
    for name, c in comm.items():
        if "reduce_scatter_kernel" in name or "all_reduce_kernel" in name or "signal_barrier" in name:
            assert _has(c, "STG.E.STRONG.SYS") and _has(c, "LDG.E.STRONG.SYS"), name   # cross-GPU flags
    assert _has(comm["b200::p2p_all_gather_kernel"], "LDG.E.NA.128")


def test_streaming_layernorm_backward_uses_bulk_copies(census):
    kernels = {k: c for k, c in census["layernorm_stream.cu.o"].items() if "ln_bwd_stream_kernel" in k}
    assert kernels
    for name, c in kernels.items():
        assert _has(c, "UBLKCP"), name                # cp.async.bulk row ring
        assert _has(c, "SYNCS"), name                 # mbarrier pipeline


def test_no_legacy_tensor_core_instructions_anywhere(census):
    for obj, kernels in census.items():
        for name, c in kernels.items():
            assert not _has(c, "HMMA"), (obj, name)   # mma.sync / wmma would show up as HMMA


def test_collective_kernels_are_light_enough_to_sit_next_to_a_gemm_cta():
    """The collectives are launched as light CTAs: no shared memory and 128 threads x <= 96 registers (csrc/comm.cu), so
    five of them fit one SM's register file.  A resident GEMM CTA leaves no room for them (224 KB of shared memory, 384 x
    168 registers); they get an SM when a GEMM CTA retires.  Overlap of collectives with GEMMs is not measured on H100."""
    import re
    import subprocess

    txt = subprocess.run(["cuobjdump", "-res-usage", os.path.join(BUILD, "comm.cu.o")], capture_output=True,
                         text=True).stdout
    rows = re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)", txt)
    assert len(rows) >= 10
    for name, reg, shared in rows:
        assert int(reg) <= 96 and int(shared) == 0, (name, reg, shared)
