"""All-to-all miniapp for one-process-per-GPU runs (torchrun): the Python twin of ``bin/alltoall``
(csrc/miniapps/alltoall.cu).

Every rank holds a send and a receive buffer of P blocks of ``block_bytes``; after one all-to-all block p of rank r's
receive buffer is block r of rank p's send buffer (↔ MPI_Alltoall, ncclAllToAll, all_to_all_single).  Algorithms:

  push   one launch per rank: my send block q is stored into slot ``rank`` of rank q's receive buffer (default)
  pull   one launch per rank: slot ``rank`` of rank p's send buffer is loaded into my receive block p
  nccl   torch.distributed.all_to_all_single — the stock baseline

Check: before every iteration send block q of rank r gets the seeded pattern of (r, q) and the iteration, the receive
buffer a poison seed no pair uses; after the last iteration every receive block p of rank r is checked against the
seed of (p, r).  ``VirtualAlltoall`` drives ``world`` ranks from one process on one GPU.
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import List, Optional

import torch

from .. import native
from ..ops.alltoall import all_to_all, as_blocks, check_args
from ..parallel.comm import Comm
from ..parallel.symmetric import SignalPads, SymmetricBuffer

ALGOS = ("push", "pull", "nccl")
VIRTUAL_ALGOS = ("push", "pull")
POISON_SEED = 0xC0DE0000


def pair_seed(it: int, src: int, dst: int) -> int:
    """The pattern seed of block ``dst`` of rank ``src``'s send buffer in iteration ``it`` (never the poison)."""
    return 0x40000000 | ((it & 0x3FFFFF) << 8) | (src << 4) | dst


@dataclass
class AlltoallResult:
    variant: str
    world: int
    block_bytes: int
    ms: float
    mismatches: int
    ctas: int = 0

    def row(self) -> dict:
        """One JSON row with the CLI's keys; GB/s counts the P-1 blocks that leave the rank."""
        sent = float(self.world - 1) * self.block_bytes
        gbps = sent / (self.ms * 1e-3) / 1e9 if self.ms > 0 else 0.0
        return {"pattern": "alltoall", "variant": self.variant, "ranks": self.world, "block_bytes": self.block_bytes,
                "ms": self.ms, "GBps_sent_per_rank": gbps, "ctas": self.ctas, "mismatches": self.mismatches}


class AlltoallMiniapp:
    def __init__(self, comm: Comm, device: int, block_bytes: int = 16 << 20, algo: str = "push", ctas: int = 0,
                 timeout_s: float = 30.0, _shared: Optional[dict] = None):
        """``_shared``: buffers made by an in-process group (``VirtualAlltoall``): ``pads``, ``send``, ``recv``."""
        if algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}")
        check_args(comm.world, block_bytes)
        if _shared is not None and algo not in VIRTUAL_ALGOS:
            raise ValueError(f"virtual ranks run {VIRTUAL_ALGOS}: {algo} needs one process per GPU")
        self.C = native()
        self.comm, self.device = comm, device
        self.rank, self.world = comm.rank, comm.world
        self.algo, self.block_bytes, self.ctas = algo, int(block_bytes), ctas
        self.nbytes = self.world * self.block_bytes
        self.generation = 0           # iterations initialised so far: the pattern seeds of the last one are checked
        self.launch_ctas = 0
        torch.cuda.set_device(device)
        if _shared is not None:
            self.pads, self.send, self.recv = _shared["pads"], _shared["send"], _shared["recv"]
        else:
            self.pads = SignalPads(comm, device, timeout_s=timeout_s)
            self.send = SymmetricBuffer(comm, self.nbytes, device, zero=False)
            self.recv = SymmetricBuffer(comm, self.nbytes, device, zero=False)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def initialize(self) -> None:
        """Send block q <- the pattern of (rank, q) in a new iteration; the receive buffer <- the poison."""
        st, B = self._stream(), self.block_bytes
        for q in range(self.world):
            self.C.fill_pattern(self.send.local_ptr + q * B, B // 4, pair_seed(self.generation, self.rank, q), st)
        self.C.fill_pattern(self.recv.local_ptr, self.nbytes // 4, POISON_SEED, st)
        self.generation += 1

    def run_once(self) -> None:
        """Enqueue one all-to-all on the current stream.  Precondition: every rank's send buffer is final and no rank
        still reads its receive buffer (``run()`` puts ``pads.device_barrier`` before it)."""
        pads, st = self.pads, self._stream()
        if self.algo == "nccl":
            import torch.distributed as dist
            src, dst = self.send.tensor(), self.recv.tensor()
            if self.world > 1:
                dist.all_to_all_single(dst, src)
            else:
                dst.copy_(src)
            return
        pads.barrier_epoch += 1
        self.launch_ctas = all_to_all(self.send.ptrs, self.recv.ptrs, pads.buf.ptrs, pads.ticket_ptr,
                                      pads.ticket_issued, self.rank, self.block_bytes, pads.barrier_epoch,
                                      pads.timeout_ns, pads.status_ptr, self.ctas, self.device, st,
                                      self.algo == "pull")
        pads.advance_tickets(self.launch_ctas)

    def mismatches(self) -> int:
        """Wrong words of the receive buffer against the last initialised iteration: block p must be (p, rank)'s."""
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        st, B = self._stream(), self.block_bytes
        for p in range(self.world):
            self.C.verify_pattern(self.recv.local_ptr + p * B, B // 4, pair_seed(self.generation - 1, p, self.rank),
                                  count.data_ptr(), stream=st)
        torch.cuda.synchronize(self.device)
        return int(count.item())

    def run(self, iters: int = 5, warmup: int = 1) -> AlltoallResult:
        stream = torch.cuda.current_stream(self.device)
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        best = float("inf")
        for it in range(warmup + iters):
            self.initialize()
            torch.cuda.synchronize(self.device)
            self.comm.barrier()
            self.pads.device_barrier(stream.cuda_stream)
            e0.record(stream)
            self.run_once()
            e1.record(stream)
            stream.synchronize()
            self.pads.check()
            t = self.comm.max(e0.elapsed_time(e1))
            if it >= warmup:
                best = min(best, t)
        bad = self.mismatches()
        total_bad = int(self.comm.sum(bad))
        print(f"Passed {self.rank}" if bad == 0 else f"FAILED {self.rank}: {bad} wrong words", flush=True)
        return AlltoallResult(self.algo, self.world, self.block_bytes, best, total_bad, self.launch_ctas)

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        self.send.close()
        self.recv.close()
        self.pads.close()


class VirtualAlltoall:
    """``world`` AlltoallMiniapp ranks driven by ONE process on one GPU, as ``VirtualAllreduce`` does: the peer
    pointers are plain pointers, and ``run_once()`` enqueues one all-to-all per rank, each on its own stream.  Every
    rank's grid ends in the node barrier, so the grids are kept co-resident: at most ``sms // world`` CTAs each.  At
    most 8 ranks: more streams than the device's hardware queues would serialise the spinning kernels."""

    MAX_WORLD = 8

    def __init__(self, world: int, block_bytes: int, algo: str = "push", ctas: int = 0, device: int = 0,
                 timeout_s: float = 10.0):
        from ..parallel.local import LocalGroup

        if not 1 <= world <= self.MAX_WORLD:
            raise ValueError(f"virtual ranks: 1 <= world <= {self.MAX_WORLD}")
        if algo not in VIRTUAL_ALGOS:
            raise ValueError(f"virtual ranks run {VIRTUAL_ALGOS}")
        check_args(world, block_bytes)
        C = native()
        cap = max(1, C.sm_count(device) // world)
        self.ctas = min(ctas, cap) if ctas > 0 else cap
        self.world, self.block_bytes, self.device = world, int(block_bytes), device
        self.group = LocalGroup(world, [device] * world)
        pads = self.group.pads(timeout_s=timeout_s)
        send = self.group.symmetric(world * self.block_bytes, zero=False)
        recv = self.group.symmetric(world * self.block_bytes, zero=False)
        self.ranks: List[AlltoallMiniapp] = [
            AlltoallMiniapp(self.group.comms[r], device, self.block_bytes, algo, ctas=self.ctas, timeout_s=timeout_s,
                            _shared={"pads": pads[r], "send": send[r], "recv": recv[r]})
            for r in range(world)]
        self.streams = [torch.cuda.Stream(device) for _ in range(world)]

    def load(self, sends: List[torch.Tensor]) -> None:
        """Send buffer of rank r <- ``sends[r]``: a [P, B] uint8 tensor, or any tensor of P*B bytes (viewed as bytes)."""
        if len(sends) != self.world:
            raise ValueError(f"one send tensor per rank ({self.world})")
        torch.cuda.synchronize(self.device)
        for app, s in zip(self.ranks, sends):
            b = as_blocks(s, self.world)
            if b.shape[1] != self.block_bytes:
                raise ValueError(f"a send tensor must hold {self.world} x {self.block_bytes} bytes")
            app.send.tensor().copy_(b.reshape(-1))
        torch.cuda.synchronize(self.device)

    def run_once(self) -> None:
        """One all-to-all: every rank's ``run_once`` on its own stream.  Call ``synchronize`` before the next one (it
        stands in for the cross-rank barrier of the precondition)."""
        for app, st in zip(self.ranks, self.streams):
            with torch.cuda.device(app.device), torch.cuda.stream(st):
                app.run_once()

    def synchronize(self) -> None:
        for st in self.streams:
            st.synchronize()
        for app in self.ranks:
            app.pads.check()

    def results(self) -> List[torch.Tensor]:
        """The receive buffer of every rank as a [P, B] uint8 tensor on the host."""
        self.synchronize()
        return [app.recv.tensor().cpu().reshape(self.world, self.block_bytes) for app in self.ranks]

    def close(self) -> None:
        for app in self.ranks:
            app.close()


def main(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200.models.alltoall [--block-bytes B] [--algo push|pull|nccl]``"""
    import argparse

    ap = argparse.ArgumentParser(prog="alltoall", add_help=True)
    ap.add_argument("--block-bytes", type=int, default=16 << 20, help="bytes per block (default 16 MiB)")
    ap.add_argument("--algo", default="push", choices=ALGOS)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ctas", type=int, default=0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args(argv)
    comm = Comm()
    app =AlltoallMiniapp(comm, comm.device, args.block_bytes, args.algo, ctas=args.ctas)
    res = app.run(args.iters, args.warmup)
    if comm.rank == 0:
        row = res.row()
        print(f"Elapsed (max over ranks, min of {args.iters}): {res.ms:.4f} ms | alltoall {args.algo} "
              f"P={comm.world} B={args.block_bytes} | {row['GBps_sent_per_rank']:.1f} GB/s sent per rank", flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps(row) + "\n")
    app.close()
    comm.close()
    return 0 if res.mismatches == 0 else 1


if __name__ == "__main__":
    raise SystemExit(main())
