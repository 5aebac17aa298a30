"""The emulated device of tests/alltoall_emu.py extended to the all-to-all-v.

``AlltoallvEmu.all_to_all_v`` has the kernel's semantics on the bound plan rules (csrc/kernels/alltoallv_plan.h through
the real extension): the launcher's refusals in the native words, the count matrix read from every rank's counts, the
verdict, recv_counts and the verdict word, the staggered walk of the packed segments (push or pull) only if the matrix
is accepted, then the node barrier.  ``fault`` plants one defect in the launch of rank ``fault_rank`` (the test's own
emulation, not the program):

  inclusive-prefix  the send offset of a segment is the inclusive prefix of its row (it starts one segment late)
  row-recv-offset   the receive offset is summed along the sender's row instead of the receiver's column
  copy-refused      a refused matrix is copied anyway
  no-recv-counts    recv_counts is never written
  short-segment     every segment loses its last 16-byte vector
  rows-below-8      the judge reads only rows 0..7 of the matrix (a count broken in row 8 or later is accepted; what it
                    then copies is kept inside the buffers, as with copy-refused)
"""
import ctypes

import numpy as np

import tests.emu_device as emu_device
from hpc_patterns_b200.models import alltoall as alltoall_mod
from hpc_patterns_b200.ops import alltoall as alltoall_ops
from tests.alltoall_emu import AlltoallEmu, AlltoallEmuNative, AlltoallSharedEmuNative, _u32

FAULTS = ("inclusive-prefix", "row-recv-offset", "copy-refused", "no-recv-counts", "short-segment", "rows-below-8")


def _i64(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_int64 * n).from_address(ptr))


class AlltoallvEmu(AlltoallEmu):
    def all_to_all_v(self, send, recv, counts, recv_counts, verdict, pads, ticket, ticket_base, rank, row_bytes,
                     send_capacity_rows, recv_capacity_rows, barrier_epoch, timeout_ns=0, status=0, ctas=0, device=0,
                     stream=0, pull=False):
        C, P, R = self.real, len(send), row_bytes
        why = C.all_to_all_v_refusal(P, R, send_capacity_rows, recv_capacity_rows)
        if why:
            raise ValueError(why)
        if not (send[rank] + send_capacity_rows * R <= recv[rank] or recv[rank] + recv_capacity_rows * R <= send[rank]):
            raise RuntimeError(C.ALL_TO_ALL_OVERLAP_ERROR)
        if not (counts[rank] + 8 * P <= recv_counts or recv_counts + 8 * P <= counts[rank]):
            raise RuntimeError(C.ALL_TO_ALL_V_COUNTS_OVERLAP_ERROR)
        m = [int(c) for p in range(P) for c in _i64(counts[p], P)]
        v = C.alltoallv_verdict(m, P, send_capacity_rows, recv_capacity_rows)
        faulty = self.fault is not None and rank == self.fault_rank
        clamp = faulty and self.fault == "copy-refused"
        if faulty and self.fault == "rows-below-8":
            clamp = v != 0
            v = C.alltoallv_verdict(m[:8 * P] + [0] * (P - 8) * P, P, send_capacity_rows, recv_capacity_rows)
        if not (faulty and self.fault == "no-recv-counts"):
            _i64(recv_counts, P)[:] = [m[p * P + rank] for p in range(P)]
        _u32(verdict).value = v
        if v == 0 or clamp:
            for j in range(P):
                p = (rank + 1 + j) % P
                s, r = (p, rank) if pull else (rank, p)
                n = m[s * P + r]
                if n <= 0:
                    continue
                src = C.alltoallv_send_offset(m, P, s, r)
                dst = C.alltoallv_recv_offset(m, P, s, r)
                nbytes = n * R
                if faulty and self.fault == "inclusive-prefix":
                    src += n
                if faulty and self.fault == "row-recv-offset":
                    dst = C.alltoallv_send_offset(m, P, r, s)
                if faulty and self.fault == "short-segment":
                    nbytes -= 16
                if clamp:                  # a kernel without the (right) verdict stays in its buffers
                    src, dst = src % send_capacity_rows, dst % recv_capacity_rows
                    n = min(n, send_capacity_rows - src, recv_capacity_rows - dst)
                    nbytes = n * R
                ctypes.memmove(recv[r] + dst * R, send[s] + src * R, nbytes)
        self._node_barrier(pads, rank, barrier_epoch)
        self.launches.append(("all_to_all_v", rank, pull))
        return self.ctas


class AlltoallvEmuNative(AlltoallvEmu, AlltoallEmuNative):
    pass


class AlltoallvSharedEmuNative(AlltoallvEmu, AlltoallSharedEmuNative):
    pass


def install(setattr_like, emu):
    """``emu_device.install`` plus the all-to-all modules."""
    emu_device.install(setattr_like, emu)
    for mod in (alltoall_mod, alltoall_ops):
        setattr_like(mod, "native", lambda: emu)


def use_in_worker(fault=None):
    """In a worker process, before the harness imports ``SharedEmuNative`` and ``install`` from tests.emu_device."""
    cls = type("FaultyAlltoallvSharedEmuNative", (AlltoallvSharedEmuNative,), {"fault": fault})
    real_install = emu_device.install
    emu_device.SharedEmuNative = cls

    def install_all(setattr_like, emu):
        real_install(setattr_like, emu)
        for mod in (alltoall_mod, alltoall_ops):
            setattr_like(mod, "native", lambda: emu)

    emu_device.install = install_all
