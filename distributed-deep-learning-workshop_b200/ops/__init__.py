"""Python entry points of the sm_90a kernels.

``ops.ext(name)`` loads (building in-tree if needed) one of the extensions:

    _b200_conv    wgmma/TMA implicit-GEMM convolution forward / dgrad / wgrad
    _b200_probe   hardware probe (TMA pipeline throughput); never on a hot path
    _b200_ops     BN / ReLU / pool / softmax-CE / preprocess kernels + fused optimizers
    _b200_comm    fused all-reduce kernels over NVLink symmetric memory
    _b200_loader  pinned-host ring buffer with side-stream H2D

On a box with a GPU the extensions are mandatory: a missing or unloadable binary raises instead of silently
falling back to eager PyTorch (``require_native``).
"""
from __future__ import annotations

from . import _build

EXT_NAMES = tuple(_build.EXTENSIONS)


# Rows per loop iteration of the BatchNorm apply / backward-apply kernels (csrc/elementwise.cu): 1, 2 or 4, bit-identical
# results; `B200DDL_BN_UNROLL` overrides the default.
BN_ROWS_UNROLL_DEFAULT = 1


def ext(name: str):
    fresh = name not in _build._loaded
    mod = _build.load(name)
    if fresh and name == "_b200_ops" and hasattr(mod, "set_bn_rows_unroll"):
        import os

        mod.set_bn_rows_unroll(int(os.environ.get("B200DDL_BN_UNROLL", BN_ROWS_UNROLL_DEFAULT)))
    return mod


def build_all(verbose: bool = False) -> None:
    _build.build_all(verbose=verbose)


def native_available() -> bool:
    import torch

    return torch.cuda.is_available()


def require_native() -> None:
    import torch

    if not torch.cuda.is_available():
        raise RuntimeError("b200ddl: this code path needs a CUDA device (H100, sm_90a)")
    cap = torch.cuda.get_device_capability()
    if cap != (9, 0):
        raise RuntimeError(f"b200ddl: kernels are compiled for sm_90a only, found sm_{cap[0]}{cap[1]}")


def kernel_launches() -> int:
    """Total number of OUR kernels launched so far (what bench.py reports as gpu_launches)."""
    import sys

    n = 0
    for name in ("_b200_ops", "_b200_comm"):
        mod = sys.modules.get(name)
        if mod is not None:
            n += int(mod.launch_count())
    from . import conv as _conv

    n += _conv.plan_launches()
    return n
