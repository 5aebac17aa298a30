"""The slab-stencil step of K-halo as a plain op on tensors (csrc/kernels/halo_stencil.cu, mode ``none``).

``stencil_step(u, lo, hi)`` computes ``alpha*u[r] + s*(u[r-1] + u[r+1])`` for the rows of one slab, with ``lo`` / ``hi``
as rows -1 / ``rows`` — the kernel the stock arm launches between its library transfers, and the compute half of the
fused step.  The exchange-carrying forms (pull / push, multi-step persistent launches, step words) live in
``hpc_patterns_b200.models.halo``; this op exists so the kernel's numerics can be checked in isolation against
``stencil_step_reference``, a plain PyTorch fp32 evaluation of the same expression, operation by operation.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import native
from ._util import current_stream, ptr


def stencil_step_reference(u: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, alpha: float = 0.5,
                           s: float = 0.25) -> torch.Tensor:
    """Plain PyTorch fp32 reference: one rounding per operation, exactly what the kernel does."""
    ext = torch.cat([lo.reshape(1, -1), u, hi.reshape(1, -1)], 0)
    a = torch.tensor(alpha, dtype=torch.float32, device=u.device)
    b = torch.tensor(s, dtype=torch.float32, device=u.device)
    return a * ext[1:-1] + b * (ext[:-2] + ext[2:])


def stencil_step(u: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor, out: Optional[torch.Tensor] = None,
                 alpha: float = 0.5, s: float = 0.25, tune: Optional[dict] = None) -> torch.Tensor:
    """``out[r] = alpha*u[r] + s*(u[r-1] + u[r+1])`` with ``u[-1] = lo``, ``u[rows] = hi`` (fp32, contiguous, row length
    a multiple of 4) through the TMA-tiled sm_90a kernel on the current stream."""
    if u.dtype != torch.float32 or u.dim() != 2 or u.shape[1] % 4:
        raise ValueError("u must be fp32 [rows, row_elems] with row_elems a multiple of 4")
    rows, row_elems = u.shape
    if lo.numel() != row_elems or hi.numel() != row_elems:
        raise ValueError("lo and hi must hold one row each")
    out = torch.empty_like(u) if out is None else out
    dev = u.device.index
    args = {"u": [ptr(u), ptr(out)], "halo_lo": [ptr(lo), ptr(lo)], "halo_hi": [ptr(hi), ptr(hi)],
            "rows": rows, "row_elems": row_elems, "alpha": alpha, "s": s, "step_base": 0, "steps": 1}
    native().halo_stencil(args, "none", dict(tune or {}), dev, current_stream(dev))
    return out
