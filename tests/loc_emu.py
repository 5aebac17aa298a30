"""The emulated device of tests/bitop_emu.py extended to maxloc / minloc on the value-index pair types.

``LocEmu`` runs ``init_pair`` / ``count_pair_mismatch`` and the loc forms of ``accumulate`` (VC = op(VC, VA)), the
default fused ring (VC a byte copy of VA at hop 0, then VC = op(VC, hop)), ``allreduce_two_shot`` (owner first) and
``ring_rsag`` (allreduce phase) on the pairs' bytes with tests/loc_oracle.py's combine.  An op that does not reduce
the type is refused with the native words (maxloc / minloc on an arithmetic type, any other op on a pair type).  Every
other case goes to ``BitOpEmu`` unchanged.  ``LocEmuNative`` is the one-process device, ``LocSharedEmuNative`` the one
for ranks in separate processes, and ``use_in_worker`` makes the multi-process harness of
tests/test_multiprocess_emulated.py build the latter.
"""
import ctypes

import numpy as np

import tests.emu_device as emu_device
from tests.bitop_emu import BitOpEmu
from tests.emu_device import _u32
from tests.lowp_emu import LowpEmuNative, LowpSharedEmuNative
from tests.loc_oracle import LAYOUT, LOC_OPS, PAIR_TYPES, combine_expected, pack, pair_bytes

_FLOAT_TYPES = ("float", "double", "bfloat16", "half")


def _refuse(op, dtype):
    """The native refusal (dtype_traits.h, reduce_op_type_error) of an op that does not reduce the type."""
    if dtype in PAIR_TYPES and op not in LOC_OPS:
        raise RuntimeError(f"op must be maxloc or minloc for {dtype}: {op} reduces arithmetic types only")
    if op in LOC_OPS and dtype not in PAIR_TYPES:
        ops = "sum, prod, min or max" if dtype in _FLOAT_TYPES else "sum, prod, min, max, band, bor, bxor, land, lor or lxor"
        raise RuntimeError(f"op must be {ops} for {dtype}: {op} reduces value-index pair types only")


def _loc(op, dtype):
    """True if (op, dtype) is a loc case; raises if one of them is loc and the other does not fit."""
    _refuse(op, dtype)
    return op in LOC_OPS


def _pair_bytes_of(value, index, dtype):
    """The pair (value, index) as the native fill writes it: the value converted to the type (static_cast)."""
    return pack((value if LAYOUT[dtype][3] else int(value), index), dtype)


class LocEmu(BitOpEmu):
    def _raw(self, ptr, n, dtype):
        return np.ctypeslib.as_array((ctypes.c_uint8 * (n * pair_bytes(dtype))).from_address(ptr))

    def _get(self, ptr, n, dtype):
        return self._raw(ptr, n, dtype).tobytes()

    def _put(self, ptr, n, dtype, b):
        self._raw(ptr, n, dtype)[:] = np.frombuffer(b, np.uint8)

    def init_pair(self, v, n, value, index, dtype, stream):
        self._put(v, n, dtype, _pair_bytes_of(value, index, dtype) * n)

    def count_pair_mismatch(self, v, n, value, index, dtype, count, stream):
        s = pair_bytes(dtype)
        got = self._raw(v, n, dtype).reshape(n, s)
        want = np.frombuffer(_pair_bytes_of(value, index, dtype), np.uint8)
        ctypes.c_int64.from_address(count).value += int((got != want).any(axis=1).sum())

    def accumulate(self, va, vc, n, dtype, stream, op="sum"):
        if not _loc(op, dtype):
            return super().accumulate(va, vc, n, dtype, stream, op)
        self._put(vc, n, dtype, combine_expected(op, self._get(vc, n, dtype), self._get(va, n, dtype), dtype))

    def ring_allreduce(self, va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n, chunk_elems,
                       epoch_base, timeout_ns, status, dtype, ctas, device, stream, slots_policy=0, ack_local=0,
                       ack_left=0, pull=False, va_left=0, slots_left=0, op="sum"):
        if not _loc(op, dtype):
            return super().ring_allreduce(va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n,
                                          chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device, stream,
                                          slots_policy, ack_local, ack_left, pull, va_left, slots_left, op)
        assert slots_policy == 0 and not pull, "the emulation covers the default ring"
        esz = pair_bytes(dtype)
        chunks = self.ring_num_chunks(n, chunk_elems, esz)
        acc = b""
        for t in range(world):
            if t > 0:
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + t, f"ring hop {t}, chunk {c}")
            src = self._get(va if t == 0 else slots_local + (t - 1) * n * esz, n, dtype)
            acc = src if t == 0 else combine_expected(op, acc, src, dtype)      # hop 0 overwrites VC
            self._put(vc, n, dtype, acc)
            if t + 1 < world:
                self._put(slots_right + t * n * esz, n, dtype, src)
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + t + 1

    def allreduce_two_shot(self, va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns, status, dtype,
                           ctas, device, stream, op="sum"):
        if not _loc(op, dtype):
            return super().allreduce_two_shot(va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns,
                                              status, dtype, ctas, device, stream, op)
        world, esz = len(va), pair_bytes(dtype)
        per = n // world
        off = rank * per * esz
        acc = self._get(va[rank] + off, per, dtype)
        for q in range(1, world):                                         # owner first
            acc = combine_expected(op, acc, self._get(va[(rank + q) % world] + off, per, dtype), dtype)
        for p in vc:
            self._put(p + off, per, dtype, acc)
        self.barrier_all(pads, rank, barrier_epoch, timeout_ns, status, stream)
        return 2

    def ring_rsag(self, va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank, world, n,
                  chunk_elems=0, epoch_base=0, timeout_ns=0, status=0, dtype="float", ctas=0, device=0, stream=0,
                  phases="allreduce", op="sum"):
        if not _loc(op, dtype):
            return super().ring_rsag(va, vc, slots_local, slots_right, vc_right, arrived_local, arrived_right, rank,
                                     world, n, chunk_elems, epoch_base, timeout_ns, status, dtype, ctas, device,
                                     stream, phases, op)
        assert phases == "allreduce", "the emulation covers the allreduce phase"
        R, ph = self.real, self.real.RSAG_ALLREDUCE
        esz = pair_bytes(dtype)
        seg_n = n // world
        chunks = self.ring_num_chunks(seg_n, chunk_elems, esz)
        for h in range(R.rsag_first_hop(ph, world), R.rsag_last_hop(ph, world) + 1):
            if R.rsag_waits(h, ph, world):
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + R.rsag_arrival(h, ph, world),
                                f"ring-rsag hop {h}, chunk {c}")
            off = R.rsag_segment(h, rank, world) * seg_n * esz
            x = self._get((vc if R.rsag_reads_vc(h, world) else va) + off, seg_n, dtype)
            rs = R.rsag_src_slot(h, ph, world)
            if rs >= 0:
                x = combine_expected(op, self._get(slots_local + rs * seg_n * esz, seg_n, dtype), x, dtype)
            if R.rsag_writes_own_vc(h, world):
                self._put(vc + off, seg_n, dtype, x)
            if R.rsag_forwards(h, ph, world):
                fs = R.rsag_fwd_slot(h, world)
                self._put(slots_right + fs * seg_n * esz if fs >= 0 else vc_right + off, seg_n, dtype, x)
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + R.rsag_arrival(h + 1, ph, world)


class LocEmuNative(LocEmu, LowpEmuNative):
    pass


class LocSharedEmuNative(LocEmu, LowpSharedEmuNative):
    pass


def use_in_worker():
    """In a worker process, before the harness imports ``SharedEmuNative`` from tests.emu_device."""
    emu_device.SharedEmuNative = LocSharedEmuNative
