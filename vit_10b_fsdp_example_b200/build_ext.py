"""In-tree build of the native extension ``vit_10b_fsdp_example_b200/_C.so``.

Every ``.cu`` file is cross-compiled for sm_90a with nvcc (works without a GPU), ``bindings.cpp`` is
compiled with g++ against the ATen headers, and everything is linked into one shared object that sits
next to the Python package so the package is importable straight from the repository tree.

    python -m vit_10b_fsdp_example_b200.build_ext [--force] [--verbose]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
BUILD_DIR = os.path.join(CSRC, "build")
SO_PATH = os.path.join(PKG_DIR, "_C.so")

CU_SOURCES = ["gemm_sm90.cu", "elementwise.cu", "comm.cu", "attention_sm90.cu", "attention_drop_sm90.cu",
              "layernorm_stream.cu", "qk_norm.cu", "layer_scale.cu", "prefix_tokens.cu",
              "patch_drop.cu", "rope.cu"]
CPP_SOURCES = ["bindings.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "--use_fast_math",
]


def _cuda_home() -> str:
    return os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _sha(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode())  # not the absolute path: the stamp must survive moving the tree
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"build step failed: {' '.join(cmd[:3])} ...")
    if verbose and (res.stdout or res.stderr):
        print(res.stdout + res.stderr)


def build(force: bool = False, verbose: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(BUILD_DIR, exist_ok=True)
    cu_sources = [s for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    all_inputs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".cpp"))]
    stamp = _sha(all_inputs) + torch.__version__
    stamp_file = os.path.join(BUILD_DIR, "stamp.txt")
    if not force and os.path.exists(SO_PATH) and os.path.exists(stamp_file):
        if open(stamp_file).read() == stamp:
            return SO_PATH

    nvcc = os.path.join(_cuda_home(), "bin", "nvcc")
    torch_inc = ce.include_paths()
    py_inc = sysconfig.get_paths()["include"]
    cuda_inc = os.path.join(_cuda_home(), "include")
    objs = []
    jobs = []
    for src in cu_sources:
        obj = os.path.join(BUILD_DIR, src + ".o")
        objs.append(obj)
        jobs.append([nvcc, *NVCC_FLAGS, "-I", CSRC, "-c", os.path.join(CSRC, src), "-o", obj])
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    for src in CPP_SOURCES:
        obj = os.path.join(BUILD_DIR, src + ".o")
        objs.append(obj)
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
               "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
               "-I", CSRC, "-I", cuda_inc, "-I", py_inc]
        for inc in torch_inc:
            cmd += ["-isystem", inc]
        cmd += ["-c", os.path.join(CSRC, src), "-o", obj]
        jobs.append(cmd)
    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        list(ex.map(lambda c: _run(c, verbose), jobs))

    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cuda_lib = os.path.join(_cuda_home(), "lib64")
    link = ["g++", "-shared", "-o", SO_PATH, *objs,
            f"-L{torch_lib}", f"-L{cuda_lib}",
            "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart",
            f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{cuda_lib}"]
    _run(link, verbose)
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return SO_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
