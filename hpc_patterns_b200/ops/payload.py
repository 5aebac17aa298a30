"""Compute payloads of the concurrency benchmark as stand-alone ops.

``busy_wait``   the dependent-FMA chain `C` (concurency/bench.hpp:23-31 maths)
``tc_busy``     the wgmma/TMA tensor-core tile loop `T` (csrc/kernels/tc_payload.cu)
``fused_group`` a whole command group as ONE persistent kernel (csrc/kernels/bench_fused.cu)
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import native
from ._util import current_stream


def busy_wait(n_items: int, tripcount: int, device: int = 0, stream: Optional[int] = None) -> torch.Tensor:
    out = torch.empty(max(n_items, 1), dtype=torch.float32, device=torch.device("cuda", device))
    native().busy_wait(out.data_ptr(), n_items, tripcount, current_stream(device) if stream is None else stream)
    return out


def busy_wait_reference(n_items: int, tripcount: int) -> torch.Tensor:
    """Closed form of the chain's result: item 0 stays 0, every other seed overflows to +inf
    once tripcount >= 1 (x, y grow doubly-exponentially over 64 dependent FMAs)."""
    ref = torch.full((max(n_items, 1),), float("inf"))
    ref[0] = 0.0
    return ref if tripcount >= 1 else torch.arange(max(n_items, 1), dtype=torch.float32)


def tc_operands(device: int = 0, stream: Optional[int] = None) -> torch.Tensor:
    C = native()
    ops = torch.zeros(C.tc_busy_operand_bytes() // 2, dtype=torch.bfloat16, device=torch.device("cuda", device))
    C.tc_fill_operands(ops.data_ptr(), current_stream(device) if stream is None else stream)
    return ops


def tc_busy(operands: torch.Tensor, ctas: int, tripcount: int, stream: Optional[int] = None,
            cluster: int = 1) -> torch.Tensor:
    """Returns out[ctas,128,256] = tripcount * (A @ B^T) computed on the tensor cores.
    ``cluster=2`` launches CTA pairs that share the B tile through TMA multicast."""
    C = native()
    dev = operands.device.index
    out = torch.empty(ctas * C.tc_busy_out_elems_per_cta(), dtype=torch.float32, device=operands.device)
    C.tc_busy(operands.data_ptr(), out.data_ptr(), ctas, tripcount,
              current_stream(dev) if stream is None else stream, cluster)
    return out.view(ctas, 128, 256)


def tc_busy_reference(operands: torch.Tensor, tripcount: int) -> torch.Tensor:
    a = operands[:128 * 64].view(128, 64).float()
    b = operands[128 * 64:].view(256, 64).float()
    return tripcount * (a @ b.t())


def fused_group(commands: List[Dict], engine: str = "tma", tune: Optional[dict] = None, device: int = 0,
                stream: Optional[int] = None) -> int:
    """Launch one fused kernel for a list of {"kind": "busy"|"triad"|"copy", ...} commands."""
    return native().fused_bench(commands, engine, tune or {}, device,
                                current_stream(device) if stream is None else stream)
