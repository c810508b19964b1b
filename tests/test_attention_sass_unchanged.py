"""The plain and the attention-dropout kernels share one kernel body per kernel (csrc/attention_sm90.cuh), instantiated
in attention_sm90.cu and attention_drop_sm90.cu.  Both objects keep the SASS, the registers and the spill bytes the
kernels had when each family had a source of its own (tests/golden/sass_before_attention_dropout_merge.json), and the
dropout object stays call-free (CPU only: nvcc and cuobjdump)."""
import json
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from helpers import sass_hash, sass_symbol_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "sass_before_attention_dropout_merge.json")
SOURCES = ["attention_sm90.cu", "attention_drop_sm90.cu"]


def _ptxas_usage(log):
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


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("cuobjdump") is None, reason="needs nvcc and cuobjdump")
def test_attention_kernels_keep_their_sass(tmp_path):
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
        assert _ptxas_usage(log) == golden["ptxas"][src], f"{src}: registers or spills changed"
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        names = {sass_symbol_key(n): n for n in re.findall(r"Function : (\S+)", sass)}
        assert sorted(names) == sorted(golden["objects"][src]), f"{src}: kernels added or gone"
        with ThreadPoolExecutor(8) as ex:
            hashes = dict(zip(names, ex.map(lambda n: sass_hash(obj, n), names.values())))
        changed = [key for key, h in golden["objects"][src].items() if hashes[key] != h]
        assert not changed, f"{src}: SASS of {len(changed)} kernels changed: {changed}"
        if src == "attention_drop_sm90.cu":  # a call would make ptxas serialise the wgmma batches (C7510)
            assert " CALL" not in sass
