"""The emulated device of tests/lowp_emu.py extended to the prod / min / max reductions (``op=``).

``OpEmu`` runs the op forms of ``accumulate`` (VC = op(VC, VA)), the default fused ring (VC overwritten at hop 0, then
VC = op(VC, hop) per hop), ``allreduce_two_shot`` (owner first; the 16-bit prod in fp32, rounded once) and
``ring_rsag`` (allreduce phase), all on raw bits with the arithmetic of tests/reduce_op_oracle.py.  ``op="sum"`` (and
no ``op``) goes to the emulation it is mixed into, unchanged.  ``OpEmuNative`` is the one-process device,
``OpSharedEmuNative`` the one for ranks in separate processes, and ``use_in_worker`` makes the multi-process harness
of tests/test_multiprocess_emulated.py build the latter.
"""
import ctypes

import numpy as np

import tests.emu_device as emu_device
from tests.emu_device import _u32
from tests.lowp_emu import LowpEmuNative, LowpSharedEmuNative
from tests.reduce_op_oracle import _UBITS, _fold, _prod16_f32, combine, elem_bytes


class OpEmu:
    def _bits(self, ptr, n, dtype):
        nb = elem_bytes(dtype)
        return np.ctypeslib.as_array((ctypes.c_uint8 * (n * nb)).from_address(ptr)).view(_UBITS[nb])

    def accumulate(self, va, vc, n, dtype, stream, op="sum"):
        if op == "sum":
            return super().accumulate(va, vc, n, dtype, stream)
        acc = self._bits(vc, n, dtype)
        acc[:] = combine(acc, self._bits(va, n, dtype), op, dtype)

    def ring_allreduce(self, va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n, chunk_elems,
                       epoch_base, timeout_ns, status, dtype, ctas, device, stream, slots_policy=0, ack_local=0,
                       ack_left=0, pull=False, va_left=0, slots_left=0, op="sum"):
        if op == "sum":
            return super().ring_allreduce(va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n,
                                          chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device, stream,
                                          slots_policy, ack_local, ack_left, pull, va_left, slots_left)
        assert slots_policy == 0 and not pull, "the emulation covers the default ring"
        esz = elem_bytes(dtype)
        chunks = self.ring_num_chunks(n, chunk_elems, esz)
        acc = self._bits(vc, n, dtype)
        for t in range(world):
            if t > 0:
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + t, f"ring hop {t}, chunk {c}")
            src = self._bits(va if t == 0 else slots_local + (t - 1) * n * esz, n, dtype)
            acc[:] = src if t == 0 else combine(acc, src, op, dtype)       # hop 0 overwrites VC
            if t + 1 < world:
                self._bits(slots_right + t * n * esz, n, dtype)[:] = src
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + t + 1

    def allreduce_two_shot(self, va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns, status, dtype,
                           ctas, device, stream, op="sum"):
        if op == "sum":
            return super().allreduce_two_shot(va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns,
                                              status, dtype, ctas, device, stream)
        world = len(va)
        per = n // world
        lo, hi = rank * per, (rank + 1) * per
        parts = [self._bits(va[(rank + q) % world], n, dtype)[lo:hi].copy() for q in range(world)]   # owner first
        total = _prod16_f32(parts, dtype) if op == "prod" and dtype in ("bfloat16", "half") else _fold(parts, op, dtype)
        for p in vc:
            self._bits(p, n, dtype)[lo:hi] = total
        self.barrier_all(pads, rank, barrier_epoch, timeout_ns, status, stream)
        return 2

    def ring_rsag(self, va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank, world, n,
                  chunk_elems=0, epoch_base=0, timeout_ns=0, status=0, dtype="float", ctas=0, device=0, stream=0,
                  phases="allreduce", op="sum"):
        if op == "sum":
            return super().ring_rsag(va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank,
                                     world, n, chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device,
                                     stream, phases)
        assert phases == "allreduce", "the emulation covers the allreduce phase"
        R, ph = self.real, self.real.RSAG_ALLREDUCE
        esz = elem_bytes(dtype)
        seg_n = n // world
        chunks = self.ring_num_chunks(seg_n, chunk_elems, esz)
        for h in range(R.rsag_first_hop(ph, world), R.rsag_last_hop(ph, world) + 1):
            if R.rsag_waits(h, ph, world):
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + R.rsag_arrival(h, ph, world),
                                f"ring-rsag hop {h}, chunk {c}")
            off = R.rsag_segment(h, rank, world) * seg_n * esz
            x = self._bits((vc if R.rsag_reads_vc(h, world) else va) + off, seg_n, dtype).copy()
            rs = R.rsag_src_slot(h, ph, world)
            if rs >= 0:
                x = combine(self._bits(slots_local + rs * seg_n * esz, seg_n, dtype), x, op, dtype)
            if R.rsag_writes_own_vc(h, world):
                self._bits(vc + off, seg_n, dtype)[:] = x
            if R.rsag_forwards(h, ph, world):
                fs = R.rsag_fwd_slot(h, world)
                self._bits(slots_right + fs * seg_n * esz if fs >= 0 else vc_right + off, seg_n, dtype)[:] = x
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + R.rsag_arrival(h + 1, ph, world)


class OpEmuNative(OpEmu, LowpEmuNative):
    pass


class OpSharedEmuNative(OpEmu, LowpSharedEmuNative):
    pass


def use_in_worker():
    """In a worker process, before the harness imports ``SharedEmuNative`` from tests.emu_device."""
    emu_device.SharedEmuNative = OpSharedEmuNative
