"""Runtime interop demos: PyTorch <-> this suite's native CUDA code.

The reference shows how two GPU runtimes (OpenMP offload and SYCL) share a device, a
context and memory, directly (``sycl_omp_ze_interopt/interop_omp_sycl.cpp:40-75``) or through
native Level-Zero handles (``interop_omp_ze_sycl.cpp:81-116``), with a cached per-device
table (``xomp_get_infos_devices`` / ``xomp_get_device_info``).  On H100 the two runtimes are
PyTorch (its caching allocator, its streams) and the raw CUDA code in ``csrc/``:

direct   * a torch tensor's ``data_ptr()`` is consumed by a native kernel, launched on
           torch's *current stream* (``torch.cuda.current_stream().cuda_stream``);
         * memory from the native allocator is viewed by torch (``__cuda_array_interface__``);
         * a native stream is adopted by torch (``torch.cuda.ExternalStream``).
native   * the driver-level handles under the runtime ordinal (CUdevice, primary CUcontext)
           and the CUcontext of torch's stream — one primary context shared by everyone;
           ownership is "keep": nothing here creates or destroys a context.

Both demos print the same progress lines as the reference and assert the data.
The torch-free native twins are ``bin/interop_torchless`` and ``bin/interop_driver``.
"""
from __future__ import annotations

from functools import lru_cache
from typing import Dict, List

import torch

from .. import native
from ..ops.p2p import pattern_reference
from ..parallel.symmetric import tensor_from_ptr


@lru_cache(maxsize=None)
def get_infos_devices() -> List[Dict]:
    """Cached table: one entry per CUDA ordinal with its native handles (↔ xomp_get_infos_devices)."""
    C = native()
    return [C.device_native_info(d) for d in range(torch.cuda.device_count())]


def get_device_info(n: int) -> Dict:
    return get_infos_devices()[n]


def demo_direct(device: int | None = None, n: int = 100, verbose: bool = True) -> None:
    C = native()
    D = torch.cuda.device_count() - 1 if device is None else device   # last device, like the reference
    torch.cuda.set_device(D)
    say = print if verbose else (lambda *a, **k: None)

    say("Torch -> HPCP")
    t = torch.full((n,), n, dtype=torch.int32, device=f"cuda:{D}")      # torch allocator + torch kernel
    say("   HPCP copy kernel using the torch pointer, on torch's current stream")
    mine = C.alloc(4 * n + 16, "D", D, True)                            # native allocator
    C.copy(mine, t.data_ptr(), 4 * n, False, "ldst", {}, {}, D, torch.cuda.current_stream(D).cuda_stream)
    view = tensor_from_ptr(mine, 4 * n, D, torch.int32)                  # torch view of native memory
    assert bool((view.cpu() == n).all()), "torch -> HPCP data mismatch"

    say("HPCP -> Torch")
    raw = C.stream_create(D, True)                                       # native stream ...
    ext = torch.cuda.ExternalStream(raw, device=D)                       # ... adopted by torch
    C.fill_pattern(mine, n, 0x1234, raw)                                 # native kernel on the native stream
    say("  Torch kernel reading the HPCP pointer, on the HPCP stream")
    with torch.cuda.stream(ext):
        out = view.to(torch.int64) & 0xFFFFFFFF                          # torch kernel, ordered after the fill
    ext.synchronize()
    assert torch.equal(out.cpu(), pattern_reference(n, 0x1234)), "HPCP -> torch data mismatch"
    del view, out
    C.stream_destroy(raw)
    C.free(mine, "D")
    say("Computation Done")


def demo_native_handles(device: int | None = None, verbose: bool = True) -> Dict:
    C = native()
    D = torch.cuda.device_count() - 1 if device is None else device
    torch.cuda.set_device(D)
    torch.zeros(1, device=f"cuda:{D}")                                   # torch has initialised the device
    info = get_device_info(D)
    stream_ctx = C.stream_context(torch.cuda.current_stream(D).cuda_stream)
    side = torch.cuda.Stream(D)
    side_ctx = C.stream_context(side.cuda_stream)
    assert stream_ctx == info["cu_context"] == side_ctx, "torch streams are not in the primary context"
    if verbose:
        print(f"Device {D}: CUdevice={info['cu_device']} primary CUcontext=0x{info['cu_context']:x} shared by "
              f"torch, the CUDA runtime and the driver API")
        print("Computation Done")
    return info
