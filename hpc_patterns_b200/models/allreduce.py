"""Allreduce miniapp for one-process-per-GPU runs (torchrun).

Capability parity with the reference miniapps
(aurora.mpich.miniapps/src/allreduce/mpi-sycl/allreduce-mpi-sycl.cpp:88-215 and the two
OpenMP variants): every rank holds VA = rank, VC = 0; after the allreduce every
element of VC equals P(P-1)/2.  Algorithms:

  ring          fused K-ring kernel: P-1 neighbour exchanges + P accumulations, one launch
  ring-unfused  the reference's step structure with separate kernels (rendezvous put, then
                accumulate), no host sync between steps
  twoshot       one-launch collective over peer mappings            (↔ MPI_Allreduce, -a)
  nvls          multimem.ld_reduce / multimem.st through torch symmetric memory's multicast
  nccl          torch.distributed.all_reduce — the stock baseline
  ring-nccl     the reference pattern verbatim through stock calls: accumulate kernel,
                NCCL send/recv, host wait, P-1 times — the baseline K-ring must beat

The native single-process CLI twin is ``bin/allreduce`` (csrc/miniapps/allreduce.cu).
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import List, Optional

import torch

from .. import native
from ..parallel.comm import Comm
from ..parallel.symmetric import SignalPads, SymmetricBuffer

ALGOS = ("ring", "ring-unfused", "twoshot", "nvls", "nccl", "ring-nccl")
# element types of the reference's datatype trait (mpi_datatype.hpp:28-51) -> the torch dtype whose add is bit-identical
# (unsigned integers share the two's-complement add of the signed type of the same width; NCCL rows only)
_TORCH_DTYPE = {"float": torch.float32, "int": torch.int32, "uint": torch.int32, "double": torch.float64,
                "long": torch.int64, "ulong": torch.int64, "short": torch.int16, "ushort": torch.int16,
                "uchar": torch.uint8}


def expected_value(world: int) -> float:
    return world * (world - 1) / 2.0


def bytes_sent_per_rank(algo: str, nbytes: int, world: int) -> float:
    """Faithful ring forwards the full block P-1 times; bandwidth-optimal collectives (P-1)/P of it."""
    if algo in ("ring", "ring-unfused", "ring-nccl"):
        return float(nbytes) * (world - 1)
    return float(nbytes) * (world - 1) / max(world, 1)


@dataclass
class AllreduceResult:
    algo: str
    dtype: str
    world: int
    elements: int
    ms: float
    mismatches: int
    elem_bytes: int = 4

    def row(self) -> dict:
        nbytes = self.elements * self.elem_bytes
        sent = bytes_sent_per_rank(self.algo, nbytes, self.world)
        gbps = sent / (self.ms * 1e-3) / 1e9 if self.ms > 0 else 0.0
        return {"pattern": "allreduce", "algo": self.algo, "type": self.dtype, "ranks": self.world,
                "elements": self.elements, "ms": self.ms, "GBps_sent_per_rank": gbps,
                "frac_of_450GBps": gbps / 450.0, "mismatches": self.mismatches}


class AllreduceMiniapp:
    def __init__(self, comm: Comm, device: int, log2_elems: int = 25, dtype: str = "float",
                 algo: str = "ring", chunk_elems: int = 0, ctas: int = 0, timeout_s: float = 30.0,
                 slots: int = 0, pull: bool = False):
        """``slots=2`` (fused ring only): two receive slots + per-chunk acks — the reference's VA/VB double
        buffer — instead of ``world-1`` slots without flow control.  ``pull=True`` (fused ring only): receiver-driven,
        every block is loaded from the left neighbour's memory instead of being stored into the right neighbour's."""
        if algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}")
        if dtype not in _TORCH_DTYPE:
            raise ValueError(f"dtype must be one of {sorted(_TORCH_DTYPE)}")
        self.C = native()
        self.comm, self.device = comm, device
        self.rank, self.world = comm.rank, comm.world
        self.algo, self.dtype, self.ctas, self.chunk_elems = algo, dtype, ctas, chunk_elems
        self.esz = self.C.elem_size(dtype)
        lanes = 16 // self.esz
        n = 1 << log2_elems
        if n % (lanes * self.world):
            n = (n // (lanes * self.world) + 1) * lanes * self.world
        self.n, self.nbytes = n, n * self.esz
        self.right, self.left = (self.rank + 1) % self.world, (self.rank - 1) % self.world
        torch.cuda.set_device(device)
        if slots not in (0, 2):
            raise ValueError("slots must be 0 (world-1 slots) or 2")
        self.slots_policy = slots if algo == "ring" else 0
        self.pull = bool(pull) and algo == "ring"
        self.n_chunks = self.C.ring_num_chunks(n, chunk_elems, self.esz)
        # arrival words, then (two-slot ring) ack words
        self.pads = SignalPads(comm, device, extra_words=self.n_chunks * (2 if self.slots_policy == 2 else 1),
                               timeout_s=timeout_s)
        self.ring_epoch = 0
        self.step_epoch = 0
        self.launches = 0
        self.va = self.vb = self.vc = self.slots = None
        self._symm = None
        if algo == "nvls":
            try:
                self._init_nvls()
            except Exception:
                self.pads.close()   # collectively allocated just above: do not leak it on the failure path
                raise
        else:
            self.va = SymmetricBuffer(comm, self.nbytes, device)
            self.vc = SymmetricBuffer(comm, self.nbytes, device)
            if algo == "ring":
                n_slots = 2 if self.slots_policy == 2 else max(self.world - 1, 1)
                self.slots = SymmetricBuffer(comm, self.nbytes * n_slots, device, zero=False)
            if algo in ("ring-unfused", "ring-nccl"):
                self.vb = SymmetricBuffer(comm, self.nbytes, device)

    # -- NVLS through torch symmetric memory (multi-process multicast mapping) -----------
    def _init_nvls(self) -> None:
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        if self.world < 2:
            raise RuntimeError("nvls needs at least 2 GPUs")
        t = symm.empty(2 * self.n, dtype=torch.float32, device=torch.device("cuda", self.device))
        hdl = symm.rendezvous(t, dist.group.WORLD)
        mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
        if mc == 0:
            raise RuntimeError("torch symmetric memory reports no multicast support on this system")
        self._symm = (t, hdl)
        self._va_ptr, self._vc_ptr = t.data_ptr(), t.data_ptr() + self.nbytes
        self._va_mc, self._vc_mc = mc, mc + self.nbytes

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _ptrs(self):
        if self.algo == "nvls":
            return self._va_ptr, self._vc_ptr
        return self.va.local_ptr, self.vc.local_ptr

    def initialize(self) -> None:
        va, vc = self._ptrs()
        vb = self.vb.local_ptr if self.vb is not None else 0
        self.C.init3(va, vb, vc, self.n, float(self.rank), float(self.rank), 0.0, self.dtype, self._stream())

    def run_once(self) -> None:
        """Enqueue one allreduce on the current stream (no host sync except for ring-nccl).

        Consecutive calls must be separated by a cross-rank barrier (``run()`` does: ``pads.device_barrier``): the
        fused ring's receive slots are reused by the next launch, and nothing inside one launch tells a rank that
        its neighbour has finished READING the previous launch's last hops."""
        C, pads, st = self.C, self.pads, self._stream()
        me, P = self.rank, self.world
        va, vc = self._ptrs()
        if self.algo == "ring":
            C.ring_allreduce(va, vc, self.slots.local_ptr, self.slots.ptrs[self.right],
                             pads.chunk_word(me), pads.chunk_word(self.right), P, self.n,
                             self.chunk_elems, self.ring_epoch, pads.timeout_ns, pads.status_ptr,
                             self.dtype, self.ctas, self.device, st, self.slots_policy,
                             pads.chunk_word(me, self.n_chunks) if self.slots_policy == 2 else 0,
                             pads.chunk_word(self.left, self.n_chunks) if self.slots_policy == 2 else 0,
                             self.pull, self.va.ptrs[self.left] if self.pull else 0,
                             self.slots.ptrs[self.left] if self.pull else 0)
            self.ring_epoch += P
            self.launches += 1
        elif self.algo == "twoshot":
            pads.barrier_epoch += 1
            ctas = C.allreduce_two_shot(self.va.ptrs, self.vc.ptrs, pads.buf.ptrs, pads.ticket_ptr,
                                        pads.ticket_issued & 0xFFFFFFFF, me, self.n, pads.barrier_epoch,
                                        pads.timeout_ns, pads.status_ptr, self.dtype, self.ctas,
                                        self.device, st)
            pads.advance_tickets(ctas)
            self.launches += 1
        elif self.algo == "nvls":
            pads.barrier_epoch += 1
            ctas = C.allreduce_nvls(self._va_mc, self._vc_mc, pads.buf.ptrs, pads.ticket_ptr,
                                    pads.ticket_issued & 0xFFFFFFFF, me, self.n, pads.barrier_epoch,
                                    pads.timeout_ns, pads.status_ptr, self.dtype, self.ctas,
                                    self.device, st)
            pads.advance_tickets(ctas)
            self.launches += 1
        elif self.algo == "nccl":
            import torch.distributed as dist
            from ..parallel.symmetric import tensor_from_ptr
            src = tensor_from_ptr(va, self.nbytes, self.device, _TORCH_DTYPE[self.dtype])
            dst = tensor_from_ptr(vc, self.nbytes, self.device, _TORCH_DTYPE[self.dtype])
            dst.copy_(src)
            if P > 1:
                dist.all_reduce(dst)
        elif self.algo == "ring-unfused":
            cur, other = va, self.vb.local_ptr
            r_other = self.vb.ptrs[self.right]
            r_cur = self.va.ptrs[self.right]
            C.accumulate(cur, vc, self.n, self.dtype, st)
            for _ in range(1, P):
                self.step_epoch += 1
                ep = self.step_epoch
                C.signal(pads.word(self.left, C.PAD_READY + me), ep, st)
                sync = pads.sync_ops(signal_rank=self.right, signal_section=C.PAD_DONE, epoch=ep,
                                     wait_section=C.PAD_READY, wait_rank=self.right)
                pads.advance_tickets(C.copy(r_other, cur, self.nbytes, False, "ldst",
                                            {"ctas": self.ctas} if self.ctas else {}, sync, self.device, st))
                C.wait(pads.word(me, C.PAD_DONE + self.left), ep, pads.timeout_ns, pads.status_ptr, st)
                cur, other = other, cur
                r_cur, r_other = r_other, r_cur
                C.accumulate(cur, vc, self.n, self.dtype, st)
                self.launches += 4
            self.launches += 1
        elif self.algo == "ring-nccl":
            import torch.distributed as dist
            from ..parallel.symmetric import tensor_from_ptr
            td = _TORCH_DTYPE[self.dtype]
            cur = tensor_from_ptr(va, self.nbytes, self.device, td)
            other = self.vb.tensor(td)
            acc = tensor_from_ptr(vc, self.nbytes, self.device, td)
            acc.add_(cur)
            torch.cuda.synchronize(self.device)        # the reference's .wait()
            for _ in range(1, P):
                ops = [dist.P2POp(dist.isend, cur, self.right), dist.P2POp(dist.irecv, other, self.left)]
                for w in dist.batch_isend_irecv(ops):
                    w.wait()
                torch.cuda.synchronize(self.device)    # blocking MPI_Send/Recv semantics
                cur, other = other, cur
                acc.add_(cur)
                torch.cuda.synchronize(self.device)

    def mismatches(self) -> int:
        _, vc = self._ptrs()
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        self.C.count_mismatch(vc, self.n, expected_value(self.world), self.dtype, count.data_ptr(),
                              self._stream())
        torch.cuda.synchronize(self.device)
        return int(count.item())

    def run(self, iters: int = 5, warmup: int = 1) -> AllreduceResult:
        stream = torch.cuda.current_stream(self.device)
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        best = float("inf")
        for it in range(warmup + iters):
            self.initialize()
            torch.cuda.synchronize(self.device)
            self.comm.barrier()
            self.pads.device_barrier(stream.cuda_stream)
            torch.cuda.nvtx.range_push(f"allreduce {self.algo} {'warm-up' if it < warmup else 'timed'}")
            e0.record(stream)
            self.run_once()
            e1.record(stream)
            torch.cuda.nvtx.range_pop()
            stream.synchronize()
            self.pads.check()
            t = self.comm.max(e0.elapsed_time(e1))
            if it >= warmup:
                best = min(best, t)
        bad = self.mismatches()
        total_bad = int(self.comm.sum(bad))
        print(f"Passed {self.rank}" if bad == 0 else f"FAILED {self.rank}: {bad} wrong elements", flush=True)
        return AllreduceResult(self.algo, self.dtype, self.world, self.n, best, total_bad, self.esz)

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        for b in (self.va, self.vb, self.vc, self.slots):
            if b is not None:
                b.close()
        self.pads.close()


def choose_collective(comm: Comm, device: int, dtype: str, log2_elems: int):
    """Which one-launch collective the ``-a`` path (↔ MPI_Allreduce, allreduce-mpi-sycl.cpp:61-67) uses.

    Decided BEFORE anything is allocated and agreed across ranks (min over ranks of the local probe), so ranks can
    neither diverge on the algorithm nor leak a half-built instance:
      * int:   two-shot — ``multimem.ld_reduce`` has no vector form for .s32 (one 4-byte request per thread), peer loads are 128-bit for every type;
      * float: NVLS (in-switch reduction) when every rank reports multicast support, else two-shot."""
    C = native()
    if dtype != "float":
        return "twoshot", "integer reductions use vector peer loads; multimem.ld_reduce.s32 is scalar"
    ok = comm.world >= 2 and bool(C.multicast_supported(device))
    if comm.min(1.0 if ok else 0.0) < 1.0:
        return "twoshot", "NVLS multicast unavailable on at least one rank"
    return "nvls", "multicast supported on every rank"


def main(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200.models.allreduce [-a] [-p k] [--algo ...]``"""
    import argparse

    ap = argparse.ArgumentParser(prog="allreduce", add_help=True)
    ap.add_argument("-a", action="store_true", help="use the one-launch collective (nvls, else twoshot)")
    ap.add_argument("-p", type=int, default=25, help="2^p elements (default 25)")
    ap.add_argument("--type", default="float", choices=sorted(_TORCH_DTYPE))
    ap.add_argument("--algo", default="ring", choices=ALGOS)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None)
    ap.add_argument("--slots", type=int, default=0, choices=(0, 2),
                    help="fused ring: 2 = two receive slots + per-chunk acks (VA/VB double buffer); "
                         "default world-1 slots")
    ap.add_argument("--pull", action="store_true",
                    help="fused ring, receiver-driven: blocks are loaded from the left neighbour (peer loads)")
    args = ap.parse_args(argv)
    comm = Comm()
    device = comm.device   # chosen before the process group was bound to it (Comm.pick_device)
    algo = args.algo
    app = None
    if args.a:
        algo, why = choose_collective(comm, device, args.type, args.p)
        if comm.rank == 0:
            print(f"# -a: {algo} ({why})", flush=True)
    app = AllreduceMiniapp(comm, device, args.p, args.type, algo, slots=args.slots, pull=args.pull)
    res = app.run(args.iters, args.warmup)
    if comm.rank == 0:
        row = res.row()
        print(f"Elapsed (max over ranks, min of {args.iters}): {res.ms:.4f} ms | {algo} {args.type} "
              f"P={comm.world} N={res.elements} | {row['GBps_sent_per_rank']:.1f} GB/s sent per rank",
              flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps(row) + "\n")
    app.close()
    comm.close()
    return 0 if res.mismatches == 0 else 1


if __name__ == "__main__":
    raise SystemExit(main())
