"""The emulated device of tests/gather_scatter_emu.py and tests/alltoallv_emu.py for serial ranks (tests/wide_world.py).

``WideWorldEmuNative`` runs the five collectives that end in the node barrier, one rank at a time as the one stream does:

* ``allreduce_two_shot`` in the kernel's order, for every (type, op) the binding takes: within slice s the main-block
  vectors (the first slice_vec // (512 U) * 512 U, U from kTwoShotShapes) fold owner first, ((VA[s] o VA[s+1]) o ...),
  and so does the tail, except the sum's (but the 16-bit floats'), which goes rank 0 first; the fold is
  tests/reduce_scatter_oracle.py's, 16-bit sums and products in fp32 rounded once;
* ``reduce_scatter``, ``all_to_all``, ``all_gather`` and ``all_to_all_v`` as their twins run them;
* the node barrier as ``grid_then_node_barrier``: the rank stores the epoch into word ``rank`` of every pad, then
  checks word t of its own, wrap-safe as ``epoch_reached``; a word not reached writes TIMEOUT into the status word (the
  one-thread driver cannot wait for a later rank);
* the CTA tickets: every launch adds its grid to the rank's ticket word.

``fault`` plants one defect in the launches of rank ``fault_rank`` (the test's own emulation, not the program); the
twins' faults apply as well (``slot-minus-8``, ``rows-below-8``):

  first-8        two-shot and reduce-scatter fold only the first 8 ranks of the owner-first order
  boundary-u2    two-shot puts its main / tail boundary at U = 2 instead of the kernel's U
  word-mod-8     the rank arrives in barrier word ``rank % 8`` instead of ``rank``
  never-arrives  the rank stores no barrier word
"""
import ctypes

import numpy as np
import torch

import tests.reduce_op_oracle as rop
from tests.allreduce_oracle import two_shot_main_vectors, two_shot_u
from tests.alltoallv_emu import AlltoallvEmu
from tests.emu_device import _u32
from tests.gather_scatter_emu import GatherScatterEmu, install  # noqa: F401  (install: re-exported)
from tests.loc_emu import LocEmu
from tests.loc_oracle import PAIR_TYPES, pair_bytes
from tests.alltoall_emu import AlltoallEmuNative
from tests.lowp_emu import LowpEmuNative
from tests.reduce_scatter_oracle import fold

FAULTS = ("first-8", "boundary-u2", "word-mod-8", "never-arrives")
LOWP = ("bfloat16", "half")


def _reached(seen, want):
    return (seen - want) & 0xFFFFFFFF < 1 << 31


class WideWorldEmu:
    fault = None
    fault_rank = 1

    def _hit(self, fault, rank):
        return self.fault == fault and rank == self.fault_rank

    def _esz(self, dtype):
        return pair_bytes(dtype) if dtype in PAIR_TYPES else self.real.elem_size(dtype)

    def _fold(self, bufs, order, off, nbytes, op, dtype):
        """The bytes of ((bufs[order[0]] o bufs[order[1]]) o ...) over [off, off + nbytes)."""
        raw = [np.ctypeslib.as_array((ctypes.c_uint8 * nbytes).from_address(bufs[p] + off)).copy() for p in order]
        if dtype in PAIR_TYPES:
            return fold([r.tobytes() for r in raw], op, dtype)
        return fold([torch.from_numpy(r).view(rop.TORCH_DTYPE[dtype]) for r in raw], op,
                    dtype).contiguous().view(torch.uint8).numpy().tobytes()

    def _issued(self, ticket, grid):
        _u32(ticket).value = (_u32(ticket).value + grid) & 0xFFFFFFFF
        return grid

    def _node_barrier(self, pads, rank, epoch):
        B = self.real.PAD_BARRIER
        if not self._hit("never-arrives", rank):
            word = rank % 8 if self._hit("word-mod-8", rank) else rank
            for p in pads:
                _u32(p + 4 * (B + word)).value = epoch
        if not all(_reached(_u32(pads[rank] + 4 * (B + t)).value, epoch) for t in range(len(pads))):
            _u32(self._status).value = self.real.STATUS_TIMEOUT

    def allreduce_two_shot(self, va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns=0, status=0,
                           dtype="float", ctas=0, device=0, stream=0, op="sum"):
        op = "prod" if op == "product" else op
        P = len(va)
        sb = n // P * self._esz(dtype)
        main = two_shot_main_vectors(sb // 16, P, 2 if self._hit("boundary-u2", rank) else two_shot_u(P)) * 16
        order = [(rank + q) % P for q in range(P)]
        if self._hit("first-8", rank):
            order = order[:8]
        tail_order = sorted(order) if op == "sum" and dtype not in LOWP else order   # kOwnerFirstTail
        out = b"".join(self._fold(va, o, rank * sb + lo, hi - lo, op, dtype)
                       for o, lo, hi in ((order, 0, main), (tail_order, main, sb)) if hi > lo)
        for p in vc:
            ctypes.memmove(p + rank * sb, out, sb)
        self._status = status
        self._node_barrier(pads, rank, barrier_epoch)
        return self._issued(ticket, ctas or self.ctas)

    def reduce_scatter(self, send, recv, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns=0, status=0,
                       dtype="float", ctas=0, device=0, stream=0, op="sum"):
        self._status = status
        grid = super().reduce_scatter(send, recv, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns,
                                      status, dtype, ctas, device, stream, op)
        if self._hit("first-8", rank):
            P, sb = len(send), n * self._esz(dtype)
            order = [(rank + q) % P for q in range(8)]
            ctypes.memmove(recv, self._fold(send, order, rank * sb, sb, "prod" if op == "product" else op, dtype), sb)
        return self._issued(ticket, grid)

    def all_to_all(self, send, recv, pads, ticket, ticket_base, rank, block_bytes, barrier_epoch, timeout_ns=0,
                   status=0, ctas=0, device=0, stream=0, pull=False):
        self._status = status
        return self._issued(ticket, super().all_to_all(send, recv, pads, ticket, ticket_base, rank, block_bytes,
                                                        barrier_epoch, timeout_ns, status, ctas, device, stream, pull))

    def all_gather(self, send, recv, pads, ticket, ticket_base, rank, block_bytes, barrier_epoch, timeout_ns=0,
                   status=0, ctas=0, device=0, stream=0, pull=False):
        self._status = status
        return self._issued(ticket, super().all_gather(send, recv, pads, ticket, ticket_base, rank, block_bytes,
                                                        barrier_epoch, timeout_ns, status, ctas, device, stream, pull))

    def all_to_all_v(self, send, recv, counts, recv_counts, verdict, pads, ticket, ticket_base, rank, row_bytes,
                     send_capacity_rows, recv_capacity_rows, barrier_epoch, timeout_ns=0, status=0, ctas=0, device=0,
                     stream=0, pull=False):
        self._status = status
        return self._issued(ticket, super().all_to_all_v(
            send, recv, counts, recv_counts, verdict, pads, ticket, ticket_base, rank, row_bytes, send_capacity_rows,
            recv_capacity_rows, barrier_epoch, timeout_ns, status, ctas, device, stream, pull))


class WideWorldEmuNative(WideWorldEmu, GatherScatterEmu, AlltoallvEmu, LocEmu, AlltoallEmuNative, LowpEmuNative):
    pass
