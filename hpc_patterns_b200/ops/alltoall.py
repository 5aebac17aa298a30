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


# ---------------------------------------------------------------------------------------------------- all-to-all-v ----
# ``all_to_all_v`` moves rows of ``row_bytes`` with per-peer counts that live on the device (↔ MPI_Alltoallv with packed
# displacements, all_to_all_single with split sizes): rank p's int64[P] counts say how many rows it sends to every rank,
# every CTA reads the whole P x P matrix over peer memory, and the packed layouts and the verdict are the rules of
# csrc/kernels/alltoallv_plan.h.  The host never learns a count.
ROW_ERROR = "all-to-all-v: row_bytes must be a positive multiple of 16"
CAPACITY_ERROR = "all-to-all-v: the send and receive capacities must be positive"
COUNTS_OVERLAP_ERROR = "all-to-all-v: recv_counts must not overlap this rank's send counts"
# The verdicts (0 = accepted) and their words, as all_to_all_v_verdict_words says them.
VERDICT_WORDS = {1: "all-to-all-v: a count is negative",
                 2: "all-to-all-v: a rank's counts exceed the send capacity",
                 3: "all-to-all-v: the counts into a rank exceed the receive capacity"}


def check_v_args(world: int, row_bytes: int, send_capacity_rows: int, recv_capacity_rows: int) -> None:
    """ValueError with the native words if the launcher would refuse these arguments."""
    if row_bytes <= 0 or row_bytes % 16:
        raise ValueError(ROW_ERROR)
    if not 1 <= world <= MAX_RANKS:
        raise ValueError(WORLD_ERROR)
    if send_capacity_rows <= 0 or recv_capacity_rows <= 0:
        raise ValueError(CAPACITY_ERROR)


def check_verdict(verdict: int) -> None:
    """ValueError with the verdict's words unless it is 0."""
    if verdict:
        raise ValueError(VERDICT_WORDS.get(verdict, f"all-to-all-v: unknown verdict {verdict}"))


def all_to_all_v(send: Sequence[int], recv: Sequence[int], counts: Sequence[int], recv_counts: int, verdict: int,
                 pads: Sequence[int], ticket: int, ticket_base: int, rank: int, row_bytes: int,
                 send_capacity_rows: int, recv_capacity_rows: int, barrier_epoch: int, timeout_ns: int = 0,
                 status: int = 0, ctas: int = 0, device: int = 0, stream: int = 0, pull: bool = False) -> int:
    """Enqueue one all-to-all-v of rank ``rank`` on ``stream``.  ``send`` / ``recv`` / ``counts`` / ``pads`` are every
    rank's peer-mapped addresses, ``recv_counts`` (int64[P]) and ``verdict`` (one 32-bit word) this rank's.  Returns
    the CTAs launched (advance the ticket counter by it)."""
    world = len(send)
    check_v_args(world, row_bytes, send_capacity_rows, recv_capacity_rows)
    if len(recv) != world or len(counts) != world or len(pads) != world:
        raise ValueError("all-to-all-v: inconsistent rank lists")
    s, r = send[rank], recv[rank]
    if not (s + send_capacity_rows * row_bytes <= r or r + recv_capacity_rows * row_bytes <= s):
        raise ValueError(OVERLAP_ERROR)
    if not (counts[rank] + 8 * world <= recv_counts or recv_counts + 8 * world <= counts[rank]):
        raise ValueError(COUNTS_OVERLAP_ERROR)
    return native().all_to_all_v(list(send), list(recv), list(counts), recv_counts, verdict, list(pads), ticket,
                                 ticket_base & 0xFFFFFFFF, rank, row_bytes, send_capacity_rows, recv_capacity_rows,
                                 barrier_epoch, timeout_ns, status, ctas, device, stream, pull)


def all_to_all_v_reference(sends: List[torch.Tensor], counts: List, row_bytes: int) -> List[torch.Tensor]:
    """The receive rows of every rank: rank r gets, for p = 0 ... P-1, the ``counts[p][r]`` rows of rank p's send
    buffer that start at row sum(counts[p][:r]).  ``sends[p]`` is any tensor of at least sum(counts[p]) rows (viewed as
    bytes); the result is one [sum_p counts[p][r], row_bytes] uint8 tensor per rank."""
    world = len(sends)
    m = [[int(c) for c in (row.tolist() if torch.is_tensor(row) else row)] for row in counts]
    rows = [s.contiguous().view(torch.uint8).reshape(-1)[: sum(m[p]) * row_bytes].reshape(-1, row_bytes)
            for p, s in enumerate(sends)]
    out = []
    for r in range(world):
        segs = [rows[p][sum(m[p][:r]): sum(m[p][:r]) + m[p][r]] for p in range(world)]
        out.append(torch.cat(segs) if segs else torch.empty(0, row_bytes, dtype=torch.uint8))
    return out


# ------------------------------------------------------------------------------------------------------ all-gather ----
# ``all_gather`` is the one-launch all-gather (↔ MPI_Allgather, ncclAllGather, all_gather_into_tensor): every rank holds
# one send block of ``block_bytes``; afterwards block p of every rank's receive buffer (P blocks) is rank p's send block.
# It is the all-to-all's walk with a source stride of 0, push or pull, ending with the node barrier.
# Its refusal words are the native module's (csrc/kernels/api.h), read from it.


def check_gather_args(world: int, block_bytes: int) -> None:
    """ValueError with the native words if the launcher would refuse (world, block_bytes)."""
    if block_bytes <= 0 or block_bytes % 16:
        raise ValueError(native().ALL_GATHER_BLOCK_ERROR)
    if not 1 <= world <= MAX_RANKS:
        raise ValueError(native().ALL_GATHER_WORLD_ERROR)


def all_gather(send: Sequence[int], recv: Sequence[int], pads: Sequence[int], ticket: int, ticket_base: int, rank: int,
               block_bytes: int, barrier_epoch: int, timeout_ns: int = 0, status: int = 0, ctas: int = 0,
               device: int = 0, stream: int = 0, pull: bool = False) -> int:
    """Enqueue one all-gather of rank ``rank`` on ``stream``.  ``send`` / ``recv`` / ``pads`` are every rank's
    peer-mapped addresses.  Returns the CTAs launched (advance the ticket counter by it)."""
    world = len(send)
    check_gather_args(world, block_bytes)
    if len(recv) != world or len(pads) != world:
        raise ValueError("all-gather: inconsistent rank lists")
    if not 0 <= rank < world:
        raise ValueError("all-gather: rank out of range")
    s, r = send[rank], recv[rank]
    if not (s + block_bytes <= r or r + world * block_bytes <= s):
        raise ValueError(native().ALL_GATHER_OVERLAP_ERROR)
    return native().all_gather(list(send), list(recv), list(pads), ticket, ticket_base & 0xFFFFFFFF, rank, block_bytes,
                               barrier_epoch, timeout_ns, status, ctas, device, stream, pull)


def all_gather_reference(sends: List[torch.Tensor]) -> torch.Tensor:
    """The receive buffer of every rank: the bytes of ``sends[0]``, ``sends[1]``, ... concatenated, as [P, B] uint8."""
    return torch.stack([s.contiguous().view(torch.uint8).reshape(-1) for s in sends])
