"""Functional op sets: ``torch_ops`` (reference / CPU) and ``cuda_ops`` (hand-written sm_90a kernels)."""
from . import torch_ops  # noqa: F401


def get_ops(device_type: str):
    if device_type == "cuda":
        from . import cuda_ops

        return cuda_ops
    return torch_ops
