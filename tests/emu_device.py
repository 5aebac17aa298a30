"""An emulated device for the CPU tier: the surface of the native extension that the flagship's Python layer uses,
implemented on host memory.  Addresses are real host addresses, a "launch" executes at once, and the emulated
`halo_stencil` has the semantics of the kernel it stands in for (see tests/test_halo_python_emulated.py).

`EmuNative`       one process: a wait that is not satisfied yet is a deadlock of the one-thread driver -> raises.
`SharedEmuNative` several processes: allocations live in named shared-memory segments, `ipc_export` / `ipc_open` hand
                  them to the peers (the role CUDA IPC plays on the device), waits SPIN with a deadline like the device
                  code does — so ranks in different processes really run concurrently against each other's step words.
`install(setattr_like, emu)` points the package at the emulation (pytest's monkeypatch.setattr, or plain setattr in a
disposable worker process)."""
import contextlib
import ctypes
import time
from multiprocessing import shared_memory

import numpy as np
import torch

import hpc_patterns_b200
from hpc_patterns_b200.models import allreduce as allreduce_mod
from hpc_patterns_b200.models import halo as halo_mod
from hpc_patterns_b200.models import peer2pear as peer2pear_mod
from hpc_patterns_b200.models.halo import initial_field, reference_steps
from hpc_patterns_b200.parallel import local as local_mod
from hpc_patterns_b200.parallel import symmetric as symmetric_mod
from tests.field_compare import count_far, count_wrong

FLAG_WORDS = 8          # kHaloFlagWords (csrc/kernels/api.h): one 32-byte sector per CTA


def _f32(ptr, n):
    return torch.frombuffer((ctypes.c_float * n).from_address(ptr), dtype=torch.float32)


def _u32(ptr):
    return ctypes.c_uint32.from_address(ptr)


class EmuNative:
    concurrent_ranks = False

    def __init__(self, ctas=3):
        self.real = hpc_patterns_b200.native()
        self.ctas = ctas
        self.live = {}
        self.launches = []

    def __getattr__(self, name):          # constants (PAD_*, HALO_*, STATUS_*) come from the real extension
        attr = getattr(self.real, name)
        if callable(attr):
            raise AttributeError(f"EmuNative: {name} is not emulated")
        return attr

    # ---- memory ----------------------------------------------------------------------------
    def alloc(self, nbytes, kind="D", device=0, zero=True):
        buf = np.zeros(nbytes + 64, dtype=np.uint8) if zero else np.full(nbytes + 64, 0xA5, dtype=np.uint8)
        addr = (buf.ctypes.data + 63) & ~63
        self.live[addr] = buf
        return addr

    def free(self, ptr, kind="D"):
        del self.live[ptr]

    def memset_async(self, ptr, value, nbytes, stream):
        ctypes.memset(ptr, value, nbytes)

    def memcpy_async(self, dst, src, nbytes, stream):
        ctypes.memmove(dst, src, nbytes)

    def read_u32(self, ptr):
        return _u32(ptr).value

    def enable_peer_access(self, devices):
        pass

    # ---- flags -------------------------------------------------------------------------------
    def signal(self, flag, epoch, stream):
        _u32(flag).value = epoch

    def _await(self, flag, epoch, what):
        """One process: nothing else can run while a launch executes, so an unsatisfied wait never returns."""
        have = _u32(flag).value
        if have < epoch:
            raise RuntimeError(f"{what}: the word holds {have}, this launch would spin on a step nobody has enqueued")

    def wait(self, flag, epoch, timeout_ns, status, stream):
        self._await(flag, epoch, f"wait for epoch {epoch}")

    def barrier_all(self, pads, rank, epoch, timeout_ns, status, stream):
        for p in pads:
            _u32(p + 4 * (self.real.PAD_BARRIER + rank)).value = epoch
        for r in range(len(pads)):
            self._await(pads[rank] + 4 * (self.real.PAD_BARRIER + r), epoch, f"barrier epoch {epoch}, rank {r}")

    def copy(self, dst, src, nbytes, src_is_peer=False, engine="ldst", tune=None, sync=None, device=0, stream=0):
        sync = sync or {}
        if "wait_flag" in sync:
            self.wait(sync["wait_flag"], sync["wait_epoch"], 0, 0, 0)
        ctypes.memmove(dst, src, nbytes)
        if "signal_flag" in sync:
            _u32(sync["signal_flag"]).value = sync["signal_epoch"]
        return 2

    # ---- pure host helpers of the real extension ---------------------------------------------------
    def elem_size(self, name):
        return self.real.elem_size(name)

    def ring_num_chunks(self, n, chunk_elems, elem_bytes=4):
        return self.real.ring_num_chunks(n, chunk_elems, elem_bytes)

    def multicast_supported(self, device):
        return False                       # no switch to reduce in: `-a` must agree on two-shot

    # ---- peer2pear payload ---------------------------------------------------------------------------
    @staticmethod
    def _pattern(n_words, seed):
        i = np.arange(n_words, dtype=np.uint64)
        return (((i * np.uint64(2654435761)) ^ np.uint64(seed)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)

    def fill_pattern(self, dst, n_words, seed, stream):
        np.ctypeslib.as_array((ctypes.c_uint32 * n_words).from_address(dst))[:] = self._pattern(n_words, seed)

    def verify_pattern(self, data, n_words, seed, mismatch, word_sum=0, wait_flag=0, wait_epoch=0, timeout_ns=0,
                       status=0, stream=0):
        if wait_flag:
            self._await(wait_flag, wait_epoch, "verify_pattern")
        got = np.ctypeslib.as_array((ctypes.c_uint32 * n_words).from_address(data))
        ctypes.c_int64.from_address(mismatch).value += int((got != self._pattern(n_words, seed)).sum())
        if word_sum:
            ctypes.c_int64.from_address(word_sum).value += int(got.astype(np.uint64).sum())

    # ---- allreduce miniapp ---------------------------------------------------------------------------
    _NP = {"float": np.float32, "int": np.int32, "uint": np.uint32, "double": np.float64, "long": np.int64,
           "ulong": np.uint64, "short": np.int16, "ushort": np.uint16, "uchar": np.uint8}

    def _arr(self, ptr, n, dtype):
        t = self._NP[dtype]
        return np.ctypeslib.as_array((ctypes.c_uint8 * (n * np.dtype(t).itemsize)).from_address(ptr)).view(t)

    def init3(self, va, vb, vc, n, a, b, c, dtype, stream):
        for ptr, v in ((va, a), (vb, b), (vc, c)):
            if ptr:
                self._arr(ptr, n, dtype)[:] = self._NP[dtype](v)

    def accumulate(self, va, vc, n, dtype, stream):
        self._arr(vc, n, dtype)[:] += self._arr(va, n, dtype)

    def count_mismatch(self, v, n, expected, dtype, count, stream):
        ctypes.c_int64.from_address(count).value += count_far(self._arr(v, n, dtype), expected)

    def ring_allreduce(self, va, vc, slots_local, slots_right, arrived_local, arrived_right, world, n, chunk_elems,
                       epoch_base, timeout_ns, status, dtype, ctas, device, stream, slots_policy=0, ack_local=0,
                       ack_left=0, pull=False, va_left=0, slots_left=0):
        """The faithful ring of the reference in one launch, default buffering (P-1 receive slots, hop t lands in slot
        t-1): accumulate my block, forward what I hold, wait per chunk for what my left neighbour forwards."""
        assert slots_policy == 0 and not pull, "the emulation covers the default ring"
        esz = np.dtype(self._NP[dtype]).itemsize
        chunks = self.ring_num_chunks(n, chunk_elems, esz)
        acc = self._arr(vc, n, dtype)
        for t in range(world):
            if t > 0:
                for c in range(chunks):
                    self._await(arrived_local + 4 * c, epoch_base + t, f"ring hop {t}, chunk {c}")
            src = self._arr(va if t == 0 else slots_local + (t - 1) * n * esz, n, dtype)
            acc += src
            if t + 1 < world:
                self._arr(slots_right + t * n * esz, n, dtype)[:] = src
                for c in range(chunks):
                    _u32(arrived_right + 4 * c).value = epoch_base + t + 1

    def allreduce_two_shot(self, va, vc, pads, ticket, ticket_base, rank, n, barrier_epoch, timeout_ns, status, dtype,
                           ctas, device, stream):
        world = len(va)
        per = n // world
        lo, hi = rank * per, (rank + 1) * per
        total = sum(self._arr(p, n, dtype)[lo:hi].astype(self._NP[dtype]) for p in va)
        for p in vc:
            self._arr(p, n, dtype)[lo:hi] = total
        self.barrier_all(pads, rank, barrier_epoch, timeout_ns, status, stream)
        return 2

    # ---- K-halo ------------------------------------------------------------------------------
    def halo_stencil_ctas(self, row_elems, mode="pull", tune=None, device=0):
        return int((tune or {}).get("ctas") or self.ctas)

    def halo_init(self, u, halo_lo, halo_hi, rows, row_elems, rank, world, stream):
        f = initial_field(world, rows, row_elems)
        G, first = world * rows, rank * rows
        _f32(u, rows * row_elems).view(rows, row_elems).copy_(f[first:first + rows])
        if halo_lo:
            _f32(halo_lo, row_elems).copy_(f[(first + G - 1) % G])
        if halo_hi:
            _f32(halo_hi, row_elems).copy_(f[(first + rows) % G])

    def _flag(self, base, flag_set, side, cta):
        return base + 4 * ((flag_set * 2 + side) * self.real.HALO_MAX_CTAS + cta) * FLAG_WORDS

    def halo_stencil(self, a, mode="pull", tune=None, device=0, stream=0):
        tune = tune or {}
        R, n = a["rows"], a["row_elems"]
        tile = (tune.get("tile_kb") or 16) * 1024 // 4
        tiles = (n + tile - 1) // tile
        t0, t1 = a.get("tile_begin", 0), a.get("tile_end", 0) or tiles
        assert 0 <= t0 < t1 <= tiles, "bad column-tile range"
        c0, c1 = t0 * tile, min(n, t1 * tile)
        ctas = self.halo_stencil_ctas(n, mode, tune)
        alpha = torch.tensor(a["alpha"], dtype=torch.float32)
        s = torch.tensor(a["s"], dtype=torch.float32)
        fs = a.get("flag_set", 0)
        self.launches.append((mode, a["step_base"], a["steps"], t0, t1, fs))
        if mode != "none" and a["steps"] > 1 and not self.concurrent_ranks:
            own = a["left_u"][0] == a["u"][0] and a["right_u"][0] == a["u"][0]
            assert own, "one process: a multi-step launch can only run when the rank is its own neighbour"
        for g in range(a["step_base"], a["step_base"] + a["steps"]):
            i, o = g & 1, (g + 1) & 1
            if mode != "none":       # the DMA thread's wait_epoch on both neighbour words of every CTA
                for c in range(ctas):
                    for side in (0, 1):
                        self._await(self._flag(a["flags_local"], fs, side, c), g,
                                    f"step {g}, word (set {fs}, side {side}, cta {c})")
            u_in = _f32(a["u"][i], R * n).view(R, n)
            u_out = _f32(a["u"][o], R * n).view(R, n)
            if mode == "pull":
                up = _f32(a["left_u"][i], R * n).view(R, n)[R - 1]
                dn = _f32(a["right_u"][i], R * n).view(R, n)[0]
            else:
                up, dn = _f32(a["halo_lo"][i], n), _f32(a["halo_hi"][i], n)
            ext = torch.cat([up[None, c0:c1], u_in[:, c0:c1], dn[None, c0:c1]], 0)
            new = alpha * ext[1:-1] + s * (ext[:-2] + ext[2:])
            u_out[:, c0:c1] = new
            if mode == "push":
                _f32(a["left_halo_hi"][o], n)[c0:c1] = new[0]
                _f32(a["right_halo_lo"][o], n)[c0:c1] = new[R - 1]
            if mode != "none":       # st.release.sys of g + 1 on both neighbours, per CTA
                for c in range(ctas):
                    _u32(self._flag(a["flags_right"], fs, 0, c)).value = g + 1   # its wait_lo: I am its left neighbour
                    _u32(self._flag(a["flags_left"], fs, 1, c)).value = g + 1    # its wait_hi
        return ctas

    def halo_verify_from_init(self, u, rows, row_elems, rank, world, steps, alpha, s, mismatch, stream):
        want = reference_steps(initial_field(world, rows, row_elems), steps, alpha, s)[rank * rows:(rank + 1) * rows]
        got = _f32(u, rows * row_elems).view(rows, row_elems)
        ctypes.c_int64.from_address(mismatch).value += count_wrong(got, want)

    def halo_verify_step(self, u_new, u_old, up_row, dn_row, rows, row_elems, alpha, s, mismatch, stream):
        old = _f32(u_old, rows * row_elems).view(rows, row_elems)
        ext = torch.cat([_f32(up_row, row_elems)[None], old, _f32(dn_row, row_elems)[None]], 0)
        a, b = torch.tensor(alpha, dtype=torch.float32), torch.tensor(s, dtype=torch.float32)
        want = a * ext[1:-1] + b * (ext[:-2] + ext[2:])
        got = _f32(u_new, rows * row_elems).view(rows, row_elems)
        ctypes.c_int64.from_address(mismatch).value += count_wrong(got, want)


class _Stream:
    cuda_stream = 0

    def __init__(self, *a, **k):
        pass

    def synchronize(self):
        pass

    def wait_stream(self, other):
        pass

    def wait_event(self, event):
        pass


class _Event:
    def __init__(self, *a, **k):
        pass

    def record(self, stream=None):
        pass




class TickingEvent(_Event):
    """cuda.Event stand-in for timed code: every start/stop pair reports 2 ms."""

    def elapsed_time(self, other):
        return 2.0


class SharedEmuNative(EmuNative):
    """The emulated device for ranks that live in DIFFERENT processes (see the module docstring)."""
    concurrent_ranks = True
    deadline_s = 30.0

    def __init__(self, ctas=3):
        super().__init__(ctas)
        self.opened = {}

    @staticmethod
    def _addr(shm):
        return ctypes.addressof(ctypes.c_char.from_buffer(shm.buf))

    def alloc(self, nbytes, kind="D", device=0, zero=True):
        shm = shared_memory.SharedMemory(create=True, size=max(int(nbytes), 64))
        addr = self._addr(shm)
        ctypes.memset(addr, 0 if zero else 0xA5, int(nbytes))
        self.live[addr] = shm
        return addr

    def free(self, ptr, kind="D"):
        shm = self.live.pop(ptr)
        self._release(shm, unlink=True)

    @staticmethod
    def _release(shm, unlink):
        try:
            shm.close()
        except BufferError:       # ctypes / torch views of the segment may still be alive in this (disposable) process
            pass
        if unlink:
            shm.unlink()

    def ipc_export(self, ptr):
        return self.live[ptr].name.encode().ljust(64, b"\0")

    def ipc_open(self, handle):
        shm = shared_memory.SharedMemory(name=handle.rstrip(b"\0").decode())
        addr = self._addr(shm)
        self.opened[addr] = shm
        return addr

    def ipc_close(self, ptr):
        self._release(self.opened.pop(ptr), unlink=False)

    def _await(self, flag, epoch, what):
        t0 = time.monotonic()
        while _u32(flag).value < epoch:
            if time.monotonic() - t0 > self.deadline_s:
                raise RuntimeError(f"{what}: timed out, the word holds {_u32(flag).value}")
            time.sleep(0)


def install(setattr_like, emu):
    """Point the package at the emulated device: native() -> emu, torch.cuda.* -> no-ops, 'cuda' tensors -> CPU."""
    for mod in (halo_mod, local_mod, symmetric_mod, allreduce_mod, peer2pear_mod):
        setattr_like(mod, "native", lambda: emu)
    view = (lambda ptr, nbytes, device, dtype=torch.uint8:
            torch.frombuffer((ctypes.c_uint8 * nbytes).from_address(ptr), dtype=torch.uint8).view(dtype))
    setattr_like(halo_mod, "tensor_from_ptr", view)
    setattr_like(symmetric_mod, "tensor_from_ptr", view)
    for name, fake in (("set_device", lambda d=None: None), ("synchronize", lambda d=None: None),
                       ("current_stream", lambda d=None: _Stream()), ("Stream", _Stream), ("Event", _Event),
                       ("device", lambda d=None: contextlib.nullcontext()),
                       ("stream", lambda s=None: contextlib.nullcontext()), ("device_count", lambda: 1)):
        setattr_like(torch.cuda, name, fake)
    setattr_like(torch.cuda.nvtx, "range_push", lambda msg: None)
    setattr_like(torch.cuda.nvtx, "range_pop", lambda: None)
    real_zeros = torch.zeros
    setattr_like(torch, "zeros", lambda *a, **k: real_zeros(*a, **{**k, "device": "cpu"}))
    setattr_like(torch.Tensor, "pin_memory", lambda self: self)
