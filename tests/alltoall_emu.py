"""The emulated device of tests/emu_device.py extended to the all-to-all.

``AlltoallEmu.all_to_all`` has the kernel's semantics: the launcher's refusals in the native words, the staggered walk
(block j goes to peer (rank + 1 + j) % P, the local block last) as one memmove per block, push or pull, then the node
barrier.  ``fault`` plants one defect in the walk of rank ``fault_rank`` (the test's own emulation, not the program):

  misroute    the blocks for ranks 0 and 2 swap destinations (slot ``rank`` of the wrong rank)
  skip-local  the local block is never copied
  short-tail  the block for rank 0 loses its last 16-byte vector
  slot-minus-8  (9 or more ranks) push stores into slot ``rank - 8`` of every receive buffer, pull loads slot
              ``rank - 8`` of every send buffer, instead of slot ``rank``

In one process the ranks run one after another, so a rank's node barrier cannot be waited for inside its launch: the
waits are kept and checked when the status word is read (``SignalPads.check``, i.e. at the synchronize that observes
the launch).  ``AlltoallSharedEmuNative`` is the device of ranks in separate processes, whose barrier spins as the
kernel's does; ``use_in_worker`` makes the multi-process harness of tests/test_multiprocess_emulated.py build it.
"""
import ctypes

import tests.emu_device as emu_device
from hpc_patterns_b200.models import alltoall as alltoall_mod
from hpc_patterns_b200.ops import alltoall as alltoall_ops
from tests.emu_device import EmuNative, SharedEmuNative, _u32

FAULTS = ("misroute", "skip-local", "short-tail", "slot-minus-8")


class AlltoallEmu:
    fault = None
    fault_rank = 1

    def sm_count(self, device):
        return 132                  # an H100 SXM: VirtualAlltoall caps every rank's grid at sms // world

    def all_to_all(self, send, recv, pads, ticket, ticket_base, rank, block_bytes, barrier_epoch, timeout_ns=0,
                   status=0, ctas=0, device=0, stream=0, pull=False):
        world, B = len(send), block_bytes
        why = self.real.all_to_all_refusal(world, B)
        if why:
            raise ValueError(why)
        if not (send[rank] + world * B <= recv[rank] or recv[rank] + world * B <= send[rank]):
            raise RuntimeError(self.real.ALL_TO_ALL_OVERLAP_ERROR)
        faulty = self.fault is not None and rank == self.fault_rank
        slot = rank - 8 if faulty and self.fault == "slot-minus-8" else rank
        for j in range(world):
            p = (rank + 1 + j) % world
            n = B
            to = p
            if faulty and self.fault == "skip-local" and p == rank:
                continue
            if faulty and self.fault == "short-tail" and p == 0:
                n = B - 16
            if faulty and self.fault == "misroute" and p in (0, 2):
                to = 2 - p
            if pull:       # my block `to` <- slot `rank` of rank p's send
                ctypes.memmove(recv[rank] + to * B, send[p] + slot * B, n)
            else:          # slot `rank` of rank `to` <- my send block p
                ctypes.memmove(recv[to] + slot * B, send[rank] + p * B, n)
        self._node_barrier(pads, rank, barrier_epoch)
        self.launches.append(("all_to_all", rank, pull))
        return self.ctas

    def _node_barrier(self, pads, rank, epoch):
        self.barrier_all(pads, rank, epoch, 0, 0, 0)


class AlltoallEmuNative(AlltoallEmu, EmuNative):
    def __init__(self, ctas=3):
        super().__init__(ctas)
        self.pending = []

    def _node_barrier(self, pads, rank, epoch):
        for p in pads:
            _u32(p + 4 * (self.real.PAD_BARRIER + rank)).value = epoch
        self.pending += [(pads[rank] + 4 * (self.real.PAD_BARRIER + r), epoch, f"node barrier {epoch}, rank {r}")
                         for r in range(len(pads))]

    def read_u32(self, ptr):
        waits, self.pending = self.pending, []
        for flag, epoch, what in waits:
            self._await(flag, epoch, what)
        return super().read_u32(ptr)


class AlltoallSharedEmuNative(AlltoallEmu, SharedEmuNative):
    pass


def install(setattr_like, emu):
    """``emu_device.install`` plus the all-to-all modules."""
    emu_device.install(setattr_like, emu)
    for mod in (alltoall_mod, alltoall_ops):
        setattr_like(mod, "native", lambda: emu)


def use_in_worker(fault=None):
    """In a worker process, before the harness imports ``SharedEmuNative`` and ``install`` from tests.emu_device."""
    cls = type("FaultyAlltoallSharedEmuNative", (AlltoallSharedEmuNative,), {"fault": fault})
    real_install = emu_device.install
    emu_device.SharedEmuNative = cls

    def install_all(setattr_like, emu):
        real_install(setattr_like, emu)
        for mod in (alltoall_mod, alltoall_ops):
            setattr_like(mod, "native", lambda: emu)

    emu_device.install = install_all
