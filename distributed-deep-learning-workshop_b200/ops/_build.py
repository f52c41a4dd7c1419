"""In-tree build + load of the sm_90a extensions.

Every extension is compiled with ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` straight into
``csrc/build/<name>/<name>.so`` (in-tree, so the binary travels to the GPU box with the repo snapshot) and is
loaded by file path.  A content hash of the sources + flags is stored next to the ``.so``; when it matches, the
binary is imported directly with no ninja/JIT step, which keeps GPU-box start-up to a dlopen.

The reference has no native code at all (SURVEY.md §2.2); these extensions are the H100-native equivalents of
what it delegates to TF/cuDNN/Horovod/NCCL/Petastorm.
"""
from __future__ import annotations

import hashlib
import importlib.util
import os
import sys
import threading
import time
from typing import Dict, List

CSRC = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "csrc"))
BUILD_ROOT = os.path.join(CSRC, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--use_fast_math",
    "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__",
    "-U__CUDA_NO_BFLOAT16_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC"]

# name -> sources (relative to csrc/)
EXTENSIONS: Dict[str, List[str]] = {
    "_b200_conv": ["conv_igemm.cu", "conv_wgrad.cu", "stem.cu", "tmap.cpp", "conv_bind.cpp"],
    "_b200_probe": ["tma_probe.cu", "tmap.cpp", "probe_bind.cpp"],   # hardware probe, not on any hot path
    "_b200_ops": ["elementwise.cu", "head_stem.cu", "mobilenet.cu", "optim.cu", "mobilenet_bwd.cu", "augment.cu",
                  "ops_bind.cpp"],
    "_b200_comm": ["allreduce.cu", "comm_bind.cpp"],
    "_b200_loader": ["ring_loader.cpp"],
    "_b200_jpeg": ["jpeg_decode.cpp", "jpeg_resize.cu"],   # nvJPEG (library) decode + our batched resize kernel
}
# extra linker flags per extension
LDFLAGS: Dict[str, List[str]] = {
    "_b200_jpeg": ["-L/usr/local/cuda/lib64", "-lnvjpeg"],
}
# headers each extension actually includes (hashed with its sources): editing one extension's header must not
# mark the others stale
HEADERS: Dict[str, List[str]] = {
    "_b200_conv": ["ptx.cuh", "conv_igemm.cuh", "conv_params.h", "conv_api.h"],
    "_b200_probe": ["ptx.cuh", "conv_params.h", "conv_api.h"],
    "_b200_ops": ["ops_api.h", "hash.cuh", "optim_rules.cuh"],
    "_b200_comm": ["comm_api.h", "optim_rules.cuh", "ops_api.h"],
    "_b200_loader": [],
    "_b200_jpeg": [],
}

_loaded: Dict[str, object] = {}
_lock = threading.Lock()


def _hash(name: str) -> str:
    h = hashlib.sha256()
    for rel in EXTENSIONS[name] + HEADERS[name]:
        p = os.path.join(CSRC, rel)
        if os.path.exists(p):
            with open(p, "rb") as f:
                h.update(rel.encode())
                h.update(f.read())
    h.update(" ".join(NVCC_FLAGS + CXX_FLAGS + LDFLAGS.get(name, [])).encode())
    import torch

    h.update(torch.__version__.encode())
    return h.hexdigest()


def so_path(name: str) -> str:
    return os.path.join(BUILD_ROOT, name, name + ".so")


def is_built(name: str) -> bool:
    hp = so_path(name) + ".hash"
    if not (os.path.exists(so_path(name)) and os.path.exists(hp)):
        return False
    with open(hp) as f:
        return f.read().strip() == _hash(name)


def build(name: str, verbose: bool = False) -> str:
    """Compile one extension with ninja (via torch.utils.cpp_extension) into csrc/build/<name>/."""
    from torch.utils import cpp_extension

    out_dir = os.path.join(BUILD_ROOT, name)
    os.makedirs(out_dir, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in EXTENSIONS[name]]
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 4))
    cpp_extension.load(
        name=name,
        sources=srcs,
        extra_cflags=CXX_FLAGS,
        extra_cuda_cflags=NVCC_FLAGS,
        extra_include_paths=[CSRC],
        extra_ldflags=list(LDFLAGS.get(name, [])),   # a copy: cpp_extension appends the torch libraries in place
        build_directory=out_dir,
        with_cuda=True,
        is_python_module=False,  # we import by path ourselves (a CPU-only box cannot always dlopen)
        verbose=verbose,
    )
    with open(so_path(name) + ".hash", "w") as f:
        f.write(_hash(name))
    return so_path(name)


def build_all(verbose: bool = False) -> None:
    for name in EXTENSIONS:
        if not is_built(name):
            build(name, verbose=verbose)


def load(name: str):
    """Import an extension module (building it first if the in-tree binary is stale or missing)."""
    with _lock:
        if name in _loaded:
            return _loaded[name]
        if not is_built(name):
            # Never silent: a stale in-tree binary on a GPU box costs minutes of nvcc per process (this is how a
            # source/.so mismatch in a snapshot looks like a hang under a short `timeout`).
            print(f"[b200ddl] extension {name} is missing or stale (source hash != {so_path(name)}.hash); "
                  f"rebuilding with nvcc - this takes minutes", file=sys.stderr, flush=True)
            t0 = time.time()
            build(name)
            print(f"[b200ddl] rebuilt {name} in {time.time() - t0:.0f}s", file=sys.stderr, flush=True)
        import torch  # noqa: F401  (libtorch symbols must be loaded before the extension)

        spec = importlib.util.spec_from_file_location(name, so_path(name))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[name] = mod
        _loaded[name] = mod
        return mod
