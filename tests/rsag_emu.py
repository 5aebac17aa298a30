"""The reduce-scatter + all-gather ring on the emulated device of tests/emu_device.py.

``RsAgEmu`` adds ``ring_rsag`` (allreduce phase) to an emulated native module: hop by hop with the kernel's own rules
(csrc/kernels/ring_order.h, through the real extension), whole segments instead of chunks, the same arrival words and
epochs.  ``RsAgSharedEmuNative`` is ``SharedEmuNative`` with it, for ranks in separate processes;
``use_in_worker`` makes the multi-process harness of tests/test_multiprocess_emulated.py build that one.
"""
import numpy as np

import tests.emu_device as emu_device
from tests.emu_device import SharedEmuNative, _u32


class RsAgEmu:
    def rsag_epoch_advance(self, phase, world):
        return self.real.rsag_epoch_advance(phase, world)

    def ring_rsag(self, va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank, world, n,
                  chunk_elems=0, epoch_base=0, timeout_ns=0, status=0, dtype="float", ctas=0, device=0, stream=0,
                  phases="allreduce"):
        assert phases == "allreduce", "the emulation covers the allreduce phase"
        R, ph = self.real, self.real.RSAG_ALLREDUCE
        esz = np.dtype(self._NP[dtype]).itemsize
        seg_n = n // world
        chunks = self.ring_num_chunks(seg_n, chunk_elems, esz)
        for h in range(R.rsag_first_hop(ph, world), R.rsag_last_hop(ph, world) + 1):
            if R.rsag_waits(h, ph, world):
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + R.rsag_arrival(h, ph, world),
                                f"ring-rsag hop {h}, chunk {c}")
            off = R.rsag_segment(h, rank, world) * seg_n * esz
            x = self._arr((vc if R.rsag_reads_vc(h, world) else va) + off, seg_n, dtype).copy()
            rs = R.rsag_src_slot(h, ph, world)
            if rs >= 0:
                x = self._arr(slots_local + rs * seg_n * esz, seg_n, dtype) + x   # wraps like the device add
            if R.rsag_writes_own_vc(h, world):
                self._arr(vc + off, seg_n, dtype)[:] = x
            if R.rsag_forwards(h, ph, world):
                fs = R.rsag_fwd_slot(h, world)
                self._arr(slots_right + fs * seg_n * esz if fs >= 0 else vc_right + off, seg_n, dtype)[:] = x
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + R.rsag_arrival(h + 1, ph, world)


class RsAgSharedEmuNative(RsAgEmu, SharedEmuNative):
    pass


def use_in_worker():
    """In a worker process, before the harness imports ``SharedEmuNative`` from tests.emu_device."""
    emu_device.SharedEmuNative = RsAgSharedEmuNative
