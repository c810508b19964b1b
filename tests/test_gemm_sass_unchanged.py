"""The GEMM kernels (csrc/gemm_sm90.cu) and the element-wise kernels that share their activation math
(csrc/epilogue_math.cuh, used by csrc/elementwise.cu) keep the SASS, the registers and the spill bytes recorded in
tests/golden/sass_gemm_before_split.json, and the GEMM object stays call-free: a call in a wgmma kernel makes ptxas
serialise its MMAs (C7510).  CPU only: nvcc and cuobjdump."""
import json
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from helpers import ptxas_usage, sass_hash, sass_symbol_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "sass_gemm_before_split.json")
SOURCES = ["gemm_sm90.cu", "elementwise.cu"]


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("cuobjdump") is None, reason="needs nvcc and cuobjdump")
def test_gemm_and_elementwise_kernels_keep_their_sass(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    golden = json.load(open(GOLDEN))
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != golden["nvcc"]:
        pytest.skip(f"the recorded SASS is from {golden['nvcc']}, this is {ver}")

    def compile_(src):
        obj = str(tmp_path / (src + ".o"))
        res = subprocess.run([NVCC, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                              os.path.join(build_ext.CSRC, src), "-o", obj], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-2000:]
        return obj, res.stdout + res.stderr

    with ThreadPoolExecutor(len(SOURCES)) as ex:
        built = dict(zip(SOURCES, ex.map(compile_, SOURCES)))
    for src, (obj, log) in built.items():
        assert "C7510" not in log, f"{src}: a call serialises the wgmma of a kernel"
        assert ptxas_usage(log) == golden["ptxas"][src], f"{src}: registers or spills changed"
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        names = {sass_symbol_key(n): n for n in re.findall(r"Function : (\S+)", sass)}
        assert sorted(names) == sorted(golden["objects"][src]), f"{src}: kernels added or gone"
        with ThreadPoolExecutor(8) as ex:
            hashes = dict(zip(names, ex.map(lambda n: sass_hash(obj, n), names.values())))
        changed = [key for key, h in golden["objects"][src].items() if hashes[key] != h]
        assert not changed, f"{src}: SASS of {len(changed)} kernels changed: {changed}"
        if src == "gemm_sm90.cu":
            assert " CALL" not in sass
