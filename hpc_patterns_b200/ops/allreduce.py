"""Allreduce building blocks (csrc/kernels/ring_allreduce.cu) on tensors or raw addresses.

``accumulate`` is the reference's ``Accumulate`` kernel (allreduce-mpi-sycl.cpp:26-31);
``ring_allreduce`` / ``two_shot`` / ``nvls`` are the fused one-launch replacements of its
``SendRecvRing`` loop and ``MPI_Allreduce``.  The multi-rank drivers live in
``hpc_patterns_b200.models.allreduce``; these wrappers are what they (and the tests) call.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import native
from ._util import current_stream, ptr

_DTYPE_NAME = {torch.float32: "float", torch.int32: "int", torch.bfloat16: "bfloat16", torch.float16: "half"}


def dtype_name(t: torch.Tensor) -> str:
    try:
        return _DTYPE_NAME[t.dtype]
    except KeyError:
        raise TypeError(f"allreduce kernels support float32, int32, bfloat16 and float16, not {t.dtype}") from None


def accumulate(va: torch.Tensor, vc: torch.Tensor, stream: Optional[int] = None) -> torch.Tensor:
    """vc += va (in place) with the native kernel; returns vc."""
    if va.shape != vc.shape or va.dtype != vc.dtype:
        raise ValueError("va and vc must have the same shape and dtype")
    dev = vc.device.index
    native().accumulate(ptr(va), ptr(vc), vc.numel(), dtype_name(vc),
                        current_stream(dev) if stream is None else stream)
    return vc


def accumulate_reference(va: torch.Tensor, vc: torch.Tensor) -> torch.Tensor:
    """Plain PyTorch reference of the same op."""
    return vc + va


def init3(va: Optional[torch.Tensor], vb: Optional[torch.Tensor], vc: Optional[torch.Tensor],
          a: float, b: float, c: float, stream: Optional[int] = None) -> None:
    ref = next(t for t in (va, vb, vc) if t is not None)
    dev = ref.device.index
    native().init3(ptr(va) if va is not None else 0, ptr(vb) if vb is not None else 0,
                   ptr(vc) if vc is not None else 0, ref.numel(), a, b, c, dtype_name(ref),
                   current_stream(dev) if stream is None else stream)


def count_mismatch(v: torch.Tensor, expected: float, stream: Optional[int] = None) -> int:
    dev = v.device.index
    count = torch.zeros(1, dtype=torch.int64, device=v.device)
    native().count_mismatch(ptr(v), v.numel(), float(expected), dtype_name(v), count.data_ptr(),
                            current_stream(dev) if stream is None else stream)
    torch.cuda.synchronize(dev)
    return int(count.item())
