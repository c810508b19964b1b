"""The attention kernels at the tile widths 32, 48, 80, 96, 112 and 144 are in the in-tree build, once each, as wgmma
kernels fed by TMA through mbarrier pipelines, and the dropout instantiations stay call-free (cuobjdump -sass, CPU
only)."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vit_10b_fsdp_example_b200", "csrc", "build")
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sass_summary  # noqa: E402

pytestmark = pytest.mark.skipif(
    shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(BUILD, "attention_sm90.cu.o"))
    or not os.path.exists(os.path.join(BUILD, "attention_drop_sm90.cu.o")),
    reason="needs cuobjdump and the in-tree build (python -m vit_10b_fsdp_example_b200.build_ext)")

WIDTHS = [32, 48, 80, 96, 112, 144]
OBJECTS = {
    "attention_sm90.cu.o": ["attn_fwd_sm90_kernel<{w}>", "attn_bwd_sm90_kernel<{w}, 0>", "attn_bwd_sm90_kernel<{w}, 1>"],
    "attention_drop_sm90.cu.o": ["attn_fwd_drop_sm90_kernel<{w}>", "attn_bwd_drop_sm90_kernel<{w}, 0>",
                                 "attn_bwd_drop_sm90_kernel<{w}, 1>"],
}


@pytest.fixture(scope="module")
def census():
    return sass_summary.census(BUILD, list(OBJECTS))


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("obj", list(OBJECTS))
def test_new_width_kernels_use_wgmma_and_tma(census, obj, w):
    for family in OBJECTS[obj]:
        name = family.format(w=w)
        kernels = {k: c for k, c in census[obj].items() if k.endswith(name)}
        assert len(kernels) == 1, name
        for c in kernels.values():
            for prefix in ("HGMMA.64", "UTMALDG.4D", "SYNCS.PHASECHK"):
                assert any(op.startswith(prefix) for op in c), (name, prefix)


def test_dropout_object_is_call_free():
    txt = subprocess.run(["cuobjdump", "-sass", os.path.join(BUILD, "attention_drop_sm90.cu.o")], capture_output=True,
                         text=True).stdout
    assert "attn_fwd_drop_sm90_kernel" in txt
    assert " CALL" not in txt
