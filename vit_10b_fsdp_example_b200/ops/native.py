"""Loader for the in-tree native extension (``vit_10b_fsdp_example_b200/_C.so``).

The extension holds every hand-written sm_90a kernel.  It is built in-tree by
``vit_10b_fsdp_example_b200.build_ext`` so the ``.so`` travels with the repo snapshot.  On a machine
with a GPU a missing extension is a hard error (no silent PyTorch fallback on the CUDA path).
"""
from __future__ import annotations

import importlib.util
import os
import threading

_PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO_PATH = os.path.join(_PKG_DIR, "_C.so")
_lock = threading.Lock()
_mod = None
_err = None


def so_path() -> str:
    return _SO_PATH


def load(build_if_missing: bool = True):
    """Return the ``_C`` module, building it first if it does not exist yet."""
    global _mod, _err
    if _mod is not None:
        return _mod
    with _lock:
        if _mod is not None:
            return _mod
        if not os.path.exists(_SO_PATH) and build_if_missing:
            from .. import build_ext

            build_ext.build()
        if not os.path.exists(_SO_PATH):
            raise RuntimeError(
                f"native extension {_SO_PATH} is missing; run `python -m vit_10b_fsdp_example_b200.build_ext`"
            )
        import torch  # noqa: F401  (libtorch must be loaded before the extension)

        spec = importlib.util.spec_from_file_location("vit_10b_fsdp_example_b200._C", _SO_PATH)
        mod = importlib.util.module_from_spec(spec)
        try:
            spec.loader.exec_module(mod)
        except Exception as e:  # pragma: no cover - surfaced to the caller
            _err = e
            raise
        _mod = mod
        return _mod


def is_built() -> bool:
    return os.path.exists(_SO_PATH)
