"""The emulated device of tests/emu_device.py extended to the 16-bit floating types, bfloat16 and half.

numpy has no bfloat16, so ``Float16Emu`` keeps the buffers of those two types as torch views, whose CPU add is the
correctly rounded 16-bit add the ring kernels do (tests/lowp_allreduce_oracle.py), and leaves every other type to the
emulation it is mixed into.  For the 16-bit types it runs:

* ``init3`` / ``accumulate`` / ``count_mismatch`` and the default fused ring (``ring_allreduce``), one rounded add per hop;
* ``allreduce_two_shot`` with the kernel's fp32 accumulation: slice s = VA[s] + VA[s+1] + ... (ranks mod P) in fp32,
  rounded once;
* ``ring_rsag`` (allreduce phase) with the hop rules of tests/rsag_emu.py;
* ``sm_count``, so that ``VirtualAllreduce`` can size its grids.

``LowpEmuNative`` is the one-process device, ``LowpSharedEmuNative`` the one for ranks in separate processes, and
``use_in_worker`` makes the multi-process harness of tests/test_multiprocess_emulated.py build the latter.
"""
import ctypes

import torch

import tests.emu_device as emu_device
from tests.emu_device import EmuNative, SharedEmuNative, _u32
from tests.field_compare import count_far
from tests.rsag_emu import RsAgEmu

TORCH16 = {"bfloat16": torch.bfloat16, "half": torch.float16}
ESZ = 2


class Float16Emu(RsAgEmu):
    def sm_count(self, device=0):
        return 132

    def _arr(self, ptr, n, dtype):
        if dtype not in TORCH16:
            return super()._arr(ptr, n, dtype)
        return torch.frombuffer((ctypes.c_uint8 * (ESZ * n)).from_address(ptr), dtype=torch.uint8).view(TORCH16[dtype])

    def init3(self, va, vb, vc, n, a, b, c, dtype, stream):
        if dtype not in TORCH16:
            return super().init3(va, vb, vc, n, a, b, c, dtype, stream)
        for ptr, v in ((va, a), (vb, b), (vc, c)):
            if ptr:
                self._arr(ptr, n, dtype)[:] = float(v)

    def count_mismatch(self, v, n, expected, dtype, count, stream):
        if dtype not in TORCH16:
            return super().count_mismatch(v, n, expected, dtype, count, stream)
        ctypes.c_int64.from_address(count).value += count_far(self._arr(v, n, dtype).double().numpy(), expected)

    def ring_allreduce(self, va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n, chunk_elems,
                       epoch_base, timeout_ns, status, dtype, ctas, device, stream, slots_policy=0, ack_local=0,
                       ack_left=0, pull=False, va_left=0, slots_left=0):
        if dtype not in TORCH16:
            return super().ring_allreduce(va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n,
                                          chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device, stream,
                                          slots_policy, ack_local, ack_left, pull, va_left, slots_left)
        assert slots_policy == 0 and not pull, "the emulation covers the default ring"
        chunks = self.ring_num_chunks(n, chunk_elems, ESZ)
        acc = self._arr(vc, n, dtype)
        for t in range(world):
            if t > 0:
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + t, f"ring hop {t}, chunk {c}")
            src = self._arr(va if t == 0 else slots_local + (t - 1) * n * ESZ, n, dtype)
            acc += src                                                          # one rounded 16-bit add
            if t + 1 < world:
                self._arr(slots_right + t * n * ESZ, n, dtype)[:] = src
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + t + 1

    def allreduce_two_shot(self, va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns, status, dtype,
                           ctas, device, stream):
        if dtype not in TORCH16:
            return super().allreduce_two_shot(va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns,
                                              status, dtype, ctas, device, stream)
        world = len(va)
        per = n // world
        lo, hi = rank * per, (rank + 1) * per
        total = self._arr(va[rank], n, dtype)[lo:hi].float()                   # fp32, owner first, rounded once
        for q in range(1, world):
            total = total + self._arr(va[(rank + q) % world], n, dtype)[lo:hi].float()
        total = total.to(TORCH16[dtype])
        for p in vc:
            self._arr(p, n, dtype)[lo:hi] = total
        self.barrier_all(pads, rank, barrier_epoch, timeout_ns, status, stream)
        return 2

    def ring_rsag(self, va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank, world, n,
                  chunk_elems=0, epoch_base=0, timeout_ns=0, status=0, dtype="float", ctas=0, device=0, stream=0,
                  phases="allreduce"):
        if dtype not in TORCH16:
            return super().ring_rsag(va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank,
                                     world, n, chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device,
                                     stream, phases)
        assert phases == "allreduce", "the emulation covers the allreduce phase"
        R, ph = self.real, self.real.RSAG_ALLREDUCE
        seg_n = n // world
        chunks = self.ring_num_chunks(seg_n, chunk_elems, ESZ)
        for h in range(R.rsag_first_hop(ph, world), R.rsag_last_hop(ph, world) + 1):
            if R.rsag_waits(h, ph, world):
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + R.rsag_arrival(h, ph, world),
                                f"ring-rsag hop {h}, chunk {c}")
            off = R.rsag_segment(h, rank, world) * seg_n * ESZ
            x = self._arr((vc if R.rsag_reads_vc(h, world) else va) + off, seg_n, dtype).clone()
            rs = R.rsag_src_slot(h, ph, world)
            if rs >= 0:
                x = self._arr(slots_local + rs * seg_n * ESZ, seg_n, dtype) + x   # one rounded 16-bit add
            if R.rsag_writes_own_vc(h, world):
                self._arr(vc + off, seg_n, dtype)[:] = x
            if R.rsag_forwards(h, ph, world):
                fs = R.rsag_fwd_slot(h, world)
                self._arr(slots_right + fs * seg_n * ESZ if fs >= 0 else vc_right + off, seg_n, dtype)[:] = x
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + R.rsag_arrival(h + 1, ph, world)


class LowpEmuNative(Float16Emu, EmuNative):
    pass


class LowpSharedEmuNative(Float16Emu, SharedEmuNative):
    pass


def use_in_worker():
    """In a worker process, before the harness imports ``SharedEmuNative`` from tests.emu_device."""
    emu_device.SharedEmuNative = LowpSharedEmuNative
