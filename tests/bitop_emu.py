"""The emulated device of tests/op_emu.py extended to the bitwise and logical reductions (band, bor, bxor, land, lor,
lxor).

``BitOpEmu`` runs their forms of ``accumulate`` (VC = op(VC, VA)), the default fused ring (VC overwritten at hop 0),
``allreduce_two_shot`` and ``ring_rsag`` (allreduce phase) on raw bits with tests/bitop_oracle.py's ``combine``, and
refuses them for the floating types with the extension's message.  Every other op goes to ``OpEmu`` unchanged.
``BitOpEmuNative`` is the one-process device, ``BitOpSharedEmuNative`` the one for ranks in separate processes, and
``use_in_worker`` makes the multi-process harness of tests/test_multiprocess_emulated.py build the latter.
"""
import tests.emu_device as emu_device
from tests.bitop_oracle import BIT_OPS, FLOAT_TYPES, combine, fold
from tests.emu_device import _u32
from tests.lowp_emu import LowpEmuNative, LowpSharedEmuNative
from tests.op_emu import OpEmu
from tests.reduce_op_oracle import elem_bytes


def _refuse_floats(op, dtype):
    if dtype in FLOAT_TYPES:
        raise RuntimeError(f"op must be sum, prod, min or max for {dtype}: {op} reduces integer types only")


class BitOpEmu(OpEmu):
    def accumulate(self, va, vc, n, dtype, stream, op="sum"):
        if op not in BIT_OPS:
            return super().accumulate(va, vc, n, dtype, stream, op)
        _refuse_floats(op, dtype)
        acc = self._bits(vc, n, dtype)
        acc[:] = combine(acc, self._bits(va, n, dtype), op, dtype)

    def ring_allreduce(self, va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n, chunk_elems,
                       epoch_base, timeout_ns, status, dtype, ctas, device, stream, slots_policy=0, ack_local=0,
                       ack_left=0, pull=False, va_left=0, slots_left=0, op="sum"):
        if op not in BIT_OPS:
            return super().ring_allreduce(va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n,
                                          chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device, stream,
                                          slots_policy, ack_local, ack_left, pull, va_left, slots_left, op)
        _refuse_floats(op, dtype)
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
        if op not in BIT_OPS:
            return super().allreduce_two_shot(va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns,
                                              status, dtype, ctas, device, stream, op)
        _refuse_floats(op, dtype)
        world = len(va)
        per = n // world
        lo, hi = rank * per, (rank + 1) * per
        total = fold([self._bits(va[(rank + q) % world], n, dtype)[lo:hi].copy() for q in range(world)], op, dtype)
        for p in vc:
            self._bits(p, n, dtype)[lo:hi] = total
        self.barrier_all(pads, rank, barrier_epoch, timeout_ns, status, stream)
        return 2

    def ring_rsag(self, va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank, world, n,
                  chunk_elems=0, epoch_base=0, timeout_ns=0, status=0, dtype="float", ctas=0, device=0, stream=0,
                  phases="allreduce", op="sum"):
        if op not in BIT_OPS:
            return super().ring_rsag(va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank,
                                     world, n, chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device,
                                     stream, phases, op)
        _refuse_floats(op, dtype)
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


class BitOpEmuNative(BitOpEmu, LowpEmuNative):
    pass


class BitOpSharedEmuNative(BitOpEmu, LowpSharedEmuNative):
    pass


def use_in_worker():
    """In a worker process, before the harness imports ``SharedEmuNative`` from tests.emu_device."""
    emu_device.SharedEmuNative = BitOpSharedEmuNative
