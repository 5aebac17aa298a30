"""K-fused-triad-put: ``a = b + s*c`` written locally AND into a peer GPU in one kernel."""
from __future__ import annotations

from typing import Optional

import torch

from .. import native
from ._util import PtrLike, current_stream, ptr


def triad_put(a_local: PtrLike, a_peer: PtrLike, b: PtrLike, c: PtrLike, s: float, n: int, *,
              engine: str = "ldst", tune: Optional[dict] = None, sync: Optional[dict] = None,
              arrive_flag: int = 0, arrive_epoch: int = 0, device: int = 0,
              stream: Optional[int] = None) -> int:
    """Fused stream triad + NVLink put.  ``a_peer=0`` runs the plain (unfused) triad."""
    C = native()
    return C.triad_put(ptr(a_local), ptr(a_peer) if not isinstance(a_peer, int) or a_peer else 0,
                       ptr(b), ptr(c), float(s), int(n), engine, tune or {}, sync or {},
                       arrive_flag, arrive_epoch, device,
                       current_stream(device) if stream is None else stream)


def triad_reference(b: torch.Tensor, c: torch.Tensor, s: float) -> torch.Tensor:
    """Plain PyTorch fp32 reference of the op (used by the numerics tests)."""
    return b.float() + float(s) * c.float()


TRIAD_SEED = 0x7A1AD000   # kTriadSeed, csrc/kernels/payload.h


def triad_inputs_reference(n: int, rank: int):
    """CPU reference of fill_triad_inputs: w = pattern word i of seed TRIAD_SEED + rank, b[i] = w & 1023,
    c[i] = (w >> 10) & 7.  No period below 2^32 elements, so a misplaced tile changes almost every value."""
    from .p2p import pattern_reference

    w = pattern_reference(n, (TRIAD_SEED + rank) & 0xFFFFFFFF)
    b = (w & 1023).float()
    c = ((w >> 10) & 7).float()
    return b, c
