"""hpc-patterns-b200: a Hopper-native GPU-communication-pattern suite.

Same capabilities and entry points as argonne-lcf/HPC-Patterns (concurrency
bench, peer2pear, topology / tile mapping, allreduce miniapps, runtime interop),
rebuilt for 8xH100: hand-written sm_90a kernels that move data over NVLink 4 /
NVSwitch peer mappings and fuse each transfer with its adjacent compute.

Layout
  ops/       Python wrappers of the sm_90a kernels (p2p copy, fused triad+put,
             ring / two-shot / NVLS allreduce, concurrency payloads)
  parallel/  process-group plumbing: symmetric peer memory (CUDA IPC / torch
             symmetric memory), signal pads, topology, rank->device mapping
  models/    the pattern programs ("model families" of this suite): concurency,
             peer2pear, allreduce miniapp, interop demos
  utils/     timing, clocks, log parser, reports, dtype table
"""
from __future__ import annotations

import os as _os

# Kernels of this suite spin on words a peer's kernel will write.  CUDA's lazy module loading cannot finish loading a
# kernel while another kernel runs on the device, so the FIRST launch of a kernel next to a spinning one deadlocks until
# the device-side deadline (csrc/common/cuda_check.h::prefer_eager_module_loading).  Must be set before the CUDA
# context exists; an explicit user setting wins.
_os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

__version__ = "0.1.0"

_ext = None


def native():
    """Return the native extension module, building nothing implicitly.

    Fails loudly when the extension is missing: on a GPU box a silent Python
    fallback would hide that the sm_90a kernels are not the ones running.
    """
    global _ext
    if _ext is not None:
        return _ext
    try:
        import importlib

        ext = importlib.import_module("hpc_patterns_b200._C")
    except Exception as e:  # pragma: no cover - depends on the build
        raise ImportError(
            "hpc_patterns_b200._C is not built. Run `python -m hpc_patterns_b200._build` "
            f"(or `make ext`) first. Original error: {e!r}") from e
    _ext = ext
    return _ext


def native_available() -> bool:
    try:
        native()
        return True
    except ImportError:
        return False
