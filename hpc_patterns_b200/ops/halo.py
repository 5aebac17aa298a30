"""The slab-stencil step of K-halo as a plain op on tensors (csrc/kernels/halo_stencil.cu, mode ``none``).

``stencil_step(u, lo, hi)`` computes ``alpha*u[r] + s*(u[r-1] + u[r+1])`` for the rows of one slab, with ``lo`` / ``hi``
as rows -1 / ``rows`` — the kernel the stock arm launches between its library transfers, and the compute half of the
fused step.  The exchange-carrying forms (pull / push, multi-step persistent launches, step words) live in
``hpc_patterns_b200.models.halo``; this op exists so the kernel's numerics can be checked in isolation against
``stencil_step_reference``, a plain PyTorch evaluation of the same expression, operation by operation.

Field types: float32, float64, bfloat16 and float16.  The step computes in fp32 (fp64 for float64) and rounds once to
the field type; ``alpha`` and ``s`` are fp32 values (see ``hpc_patterns_b200.models.halo``).
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import native
from ..models.halo import DTYPES, _native_type, compute_dtype
from ._util import current_stream, ptr


def stencil_step_reference(u: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, alpha: float = 0.5,
                           s: float = 0.25) -> torch.Tensor:
    """Plain PyTorch reference: one rounding per operation in the compute type of ``u.dtype``, then one rounding to
    ``u.dtype`` — exactly what the kernel does."""
    ct = compute_dtype(u.dtype)
    ext = torch.cat([lo.reshape(1, -1), u, hi.reshape(1, -1)], 0).to(ct)
    a = torch.tensor(alpha, dtype=torch.float32, device=u.device).to(ct)
    b = torch.tensor(s, dtype=torch.float32, device=u.device).to(ct)
    return (a * ext[1:-1] + b * (ext[:-2] + ext[2:])).to(u.dtype)


def stencil_step(u: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, out: Optional[torch.Tensor] = None,
                 alpha: float = 0.5, s: float = 0.25, tune: Optional[dict] = None) -> torch.Tensor:
    """``out[r] = alpha*u[r] + s*(u[r-1] + u[r+1])`` with ``u[-1] = lo``, ``u[rows] = hi`` (float32, float64, bfloat16
    or float16, one dtype for all four tensors, contiguous, a row a multiple of 16 bytes) through the sm_90a K-halo
    kernel on the current stream."""
    if u.dtype not in DTYPES:
        raise ValueError(f"u must be one of {[str(d) for d in DTYPES]}, not {u.dtype}")
    if u.dim() != 2 or (u.shape[1] * u.element_size()) % 16:
        raise ValueError("u must be [rows, row_elems] with a row a multiple of 16 bytes")
    rows, row_elems = u.shape
    if lo.numel() != row_elems or hi.numel() != row_elems:
        raise ValueError("lo and hi must hold one row each")
    out = torch.empty_like(u) if out is None else out
    for name, t in (("lo", lo), ("hi", hi), ("out", out)):
        if t.dtype != u.dtype:
            raise ValueError(f"{name} is {t.dtype}, u is {u.dtype}: all four tensors must share one dtype")
    dev = u.device.index
    args = {"u": [ptr(u), ptr(out)], "halo_lo": [ptr(lo), ptr(lo)], "halo_hi": [ptr(hi), ptr(hi)],
            "rows": rows, "row_elems": row_elems, "alpha": alpha, "s": s, "step_base": 0, "steps": 1}
    native().halo_stencil(args, "none", dict(tune or {}), dev, current_stream(dev), **_native_type(u.dtype))
    return out
