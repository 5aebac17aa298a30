"""The emulated device of tests/alltoall_emu.py extended to the reduce-scatter and the all-gather.

``reduce_scatter`` has the launcher's semantics: its refusals in the native words (the op's too), then rank r's result
is the owner-first fold of segment r over every rank's send buffer (tests/reduce_scatter_oracle.py) stored into its own
receive buffer, then the node barrier.  ``all_gather`` is the all-to-all's staggered walk with a source stride of 0.
``fault`` plants one defect in rank ``fault_rank``'s launch (the test's own emulation, not the program):

  neighbour-segment   the reduce-scatter folds segment rank + 1 instead of its own
  misplace            the all-gather stores its block for rank 0 into slot rank + 1 instead of slot rank

The element types come from the loc / bitop / op / 16-bit emulations (init3, init_pair and the mismatch counts).
"""
import ctypes

import numpy as np
import torch

import tests.emu_device as emu_device
import tests.reduce_op_oracle as rop
from hpc_patterns_b200.models import allreduce as allreduce_mod
from hpc_patterns_b200.models import alltoall as alltoall_mod
from hpc_patterns_b200.ops import allreduce as allreduce_ops
from hpc_patterns_b200.ops import alltoall as alltoall_ops
from tests.alltoall_emu import AlltoallEmu, AlltoallEmuNative, AlltoallSharedEmuNative
from tests.loc_emu import LocEmu
from tests.loc_oracle import PAIR_TYPES
from tests.lowp_emu import LowpEmuNative, LowpSharedEmuNative
from tests.reduce_scatter_oracle import expected

FAULTS = ("neighbour-segment", "misplace")


def _bytes(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_uint8 * n).from_address(ptr)).copy()


class GatherScatterEmu(AlltoallEmu):
    fault = None
    fault_rank = 1

    def reduce_scatter(self, send, recv, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns=0, status=0,
                       dtype="float", ctas=0, device=0, stream=0, op="sum"):
        world = len(send)
        why = self.real.reduce_scatter_refusal(world, n, dtype, op)
        if why:
            raise ValueError(why)
        seg = n * self.real.elem_size(dtype)
        if not (send[rank] + world * seg <= recv or recv + seg <= send[rank]):
            raise RuntimeError(self.real.REDUCE_SCATTER_OVERLAP_ERROR)
        op = "prod" if op == "product" else op
        raw = [_bytes(p, world * seg) for p in send]
        sends = ([r.tobytes() for r in raw] if dtype in PAIR_TYPES
                 else [torch.from_numpy(r).view(rop.TORCH_DTYPE[dtype]) for r in raw])
        mine = (rank + 1) % world if self.fault == "neighbour-segment" and rank == self.fault_rank else rank
        want = expected(sends, mine, op, dtype)
        out = np.frombuffer(want, np.uint8) if dtype in PAIR_TYPES else want.contiguous().view(torch.uint8).numpy()
        ctypes.memmove(recv, out.ctypes.data, seg)
        self._node_barrier(pads, rank, barrier_epoch)
        self.launches.append(("reduce_scatter", rank, op))
        return self.ctas

    def all_gather(self, send, recv, pads, ticket, ticket_base, rank, block_bytes, barrier_epoch, timeout_ns=0,
                   status=0, ctas=0, device=0, stream=0, pull=False):
        world, B = len(send), block_bytes
        why = self.real.all_gather_refusal(world, B)
        if why:
            raise ValueError(why)
        if not (send[rank] + B <= recv[rank] or recv[rank] + world * B <= send[rank]):
            raise RuntimeError(self.real.ALL_GATHER_OVERLAP_ERROR)
        faulty = self.fault == "misplace" and rank == self.fault_rank
        for j in range(world):
            p = (rank + 1 + j) % world
            if pull:       # my slot p <- rank p's block
                ctypes.memmove(recv[rank] + p * B, send[p], B)
            else:          # slot `rank` of rank p <- my block
                slot = (rank + 1) % world if faulty and p == 0 else rank
                ctypes.memmove(recv[p] + slot * B, send[rank], B)
        self._node_barrier(pads, rank, barrier_epoch)
        self.launches.append(("all_gather", rank, pull))
        return self.ctas


class GatherScatterEmuNative(GatherScatterEmu, LocEmu, AlltoallEmuNative, LowpEmuNative):
    pass


class GatherScatterSharedEmuNative(GatherScatterEmu, LocEmu, AlltoallSharedEmuNative, LowpSharedEmuNative):
    pass


def install(setattr_like, emu):
    """``emu_device.install`` plus the modules of both collectives."""
    emu_device.install(setattr_like, emu)
    for mod in (alltoall_mod, alltoall_ops, allreduce_mod, allreduce_ops):
        setattr_like(mod, "native", lambda: emu)


def use_in_worker(fault=None):
    """In a worker process, before the harness imports ``SharedEmuNative`` and ``install`` from tests.emu_device."""
    cls = type("FaultyGatherScatterSharedEmuNative", (GatherScatterSharedEmuNative,), {"fault": fault})
    real_install = emu_device.install
    emu_device.SharedEmuNative = cls

    def install_all(setattr_like, emu):
        real_install(setattr_like, emu)
        for mod in (alltoall_mod, alltoall_ops, allreduce_mod, allreduce_ops):
            setattr_like(mod, "native", lambda: emu)

    emu_device.install = install_all
