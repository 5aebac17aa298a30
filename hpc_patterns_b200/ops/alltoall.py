"""All-to-all building blocks (csrc/kernels/all_to_all.cu) on raw addresses, and the torch reference.

``all_to_all`` is the one-launch equal-block all-to-all (↔ MPI_Alltoall, ncclAllToAll): every rank holds a send and
a receive buffer of P blocks of ``block_bytes``; afterwards block p of rank r's receive buffer is block r of rank p's
send buffer.  ``pull=False`` (push) stores into the peers' receive buffers, ``pull=True`` loads from their send
buffers; both end with the node barrier.  The multi-rank drivers live in ``hpc_patterns_b200.models.alltoall``.
"""
from __future__ import annotations

from typing import List, Sequence

import torch

from .. import native

# The refusals of the native launcher (csrc/kernels/api.h), word for word.
BLOCK_ERROR = "all-to-all: block_bytes must be a positive multiple of 16"
WORLD_ERROR = "all-to-all: world must be between 1 and 16 ranks"
OVERLAP_ERROR = "all-to-all: the send and receive buffers must not overlap (no in-place operation)"
MAX_RANKS = 16


def check_args(world: int, block_bytes: int) -> None:
    """ValueError with the native words if the launcher would refuse (world, block_bytes)."""
    if block_bytes <= 0 or block_bytes % 16:
        raise ValueError(BLOCK_ERROR)
    if not 1 <= world <= MAX_RANKS:
        raise ValueError(WORLD_ERROR)


def check_no_overlap(send_ptr: int, recv_ptr: int, nbytes: int) -> None:
    if not (send_ptr + nbytes <= recv_ptr or recv_ptr + nbytes <= send_ptr):
        raise ValueError(OVERLAP_ERROR)


def all_to_all(send: Sequence[int], recv: Sequence[int], pads: Sequence[int], ticket: int, ticket_base: int, rank: int,
               block_bytes: int, barrier_epoch: int, timeout_ns: int = 0, status: int = 0, ctas: int = 0,
               device: int = 0, stream: int = 0, pull: bool = False) -> int:
    """Enqueue one all-to-all of rank ``rank`` on ``stream``.  ``send`` / ``recv`` / ``pads`` are every rank's
    peer-mapped addresses.  Returns the CTAs launched (advance the ticket counter by it)."""
    check_args(len(send), block_bytes)
    if len(recv) != len(send) or len(pads) != len(send):
        raise ValueError("all-to-all: inconsistent rank lists")
    check_no_overlap(send[rank], recv[rank], block_bytes * len(send))
    return native().all_to_all(list(send), list(recv), list(pads), ticket, ticket_base & 0xFFFFFFFF, rank, block_bytes,
                               barrier_epoch, timeout_ns, status, ctas, device, stream, pull)


def as_blocks(t: torch.Tensor, world: int) -> torch.Tensor:
    """``t`` (any dtype, contiguous) as ``world`` rows of bytes: the [P, B] uint8 view the all-to-all moves."""
    return t.contiguous().view(torch.uint8).reshape(world, -1)


def all_to_all_reference(sends: List[torch.Tensor]) -> List[torch.Tensor]:
    """recv[r][p] = send[p][r] for the [P, B] byte views of every rank's send buffer."""
    world = len(sends)
    s = torch.stack([as_blocks(x, world) for x in sends])        # [src, dst, B]
    return [s[:, r].contiguous() for r in range(world)]
