"""peer2pear for one-process-per-GPU runs (torchrun), and round 1's flagship fused exchange (the flagship since
round 2 is the halo exchange of models/halo.py).

Two public classes:

``P2PBench``            the reference's benchmark (p2p/peer2pear.cpp:104-156): ranks
                        paired (2k,2k+1), unidirectional then bidirectional, 10
                        iterations / min, aggregate GB/s, same result lines.  Transports
                        ``put`` (↔ MPI_Put+fence), ``get``, ``sendrecv`` (↔ Isend/Irecv),
                        plus the stock baselines ``memcpy`` (cudaMemcpyPeerAsync) and
                        ``nccl`` (torch.distributed send/recv).
``FusedTriadExchange``  round 1's headline op: every rank computes the stream
                        triad ``a = b + s*c`` and puts ``a`` into its ring neighbour
                        in ONE kernel (csrc/kernels/fused_triad_put.cu); bench.py
                        measures it, the halo-exchange style loops use it.

The native single-process CLI twin is ``bin/peer2pear`` (csrc/p2p/peer2pear.cu).
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from .. import native
from ..parallel.comm import Comm
from ..parallel.symmetric import SignalPads, SymmetricBuffer

REFERENCE_MESSAGE_BYTES = 1179648 * 40 * 4  # 188 743 680, p2p/peer2pear.cpp:115-116


def sweep_sizes(lo: int = 1 << 10, hi: int = 1 << 30) -> List[int]:
    """1 KiB .. 1 GiB in powers of two, plus the reference's 180 MiB point."""
    sizes = []
    b = lo
    while b <= hi:
        sizes.append(b)
        b <<= 1
    sizes.append(REFERENCE_MESSAGE_BYTES)
    return sorted(set(s for s in sizes if lo <= s <= max(hi, REFERENCE_MESSAGE_BYTES)))


def bandwidth_gbps(nbytes: int, pairs: int, t_ns: float, bidirectional: bool) -> float:
    """The reference's formulas (peer2pear.cpp:138,153): aggregate over all pairs; bytes/ns == GB/s."""
    return (2.0 if bidirectional else 1.0) * nbytes * pairs / t_ns


# =====================================================================================
class FusedTriadExchange:
    """Ring exchange of a freshly computed triad, fused into one kernel per rank.

    step():  a = b + s*c   (local HBM)   and   right_neighbour.recv = a   (NVLink),
             then publish the arrival epoch on the neighbour and wait for the left
             neighbour's arrival — one launch, no NCCL / cudaMemcpy / host sync.
    With world == 1 the neighbour is the rank itself (loop-back through local HBM).
    """

    def __init__(self, comm: Comm, device: int, nbytes: int = REFERENCE_MESSAGE_BYTES, s: float = 3.0,
                 engine: str = "ldst", tune: Optional[dict] = None, timeout_s: float = 30.0,
                 compute_ratio: int = 1):
        """``compute_ratio`` R: the triad runs over R x the message (the local domain) and only the
        first ``nbytes`` of the result (the halo) are put to the neighbour.  R balances the HBM time of
        the compute against the NVLink time of the put, like the reference's autotuner balances the
        commands of a group; R = 1 puts everything that is computed."""
        if nbytes % 16:
            raise ValueError("message size must be a multiple of 16 bytes")
        if compute_ratio < 1:
            raise ValueError("compute_ratio must be >= 1")
        if compute_ratio > 1 and nbytes % (16 << 10):
            raise ValueError("halo mode needs a message size that is a multiple of 16 KiB")
        self.compute_ratio = int(compute_ratio)
        self.C = native()
        self.comm, self.device = comm, device
        self.rank, self.world = comm.rank, comm.world
        self.nbytes, self.n = int(nbytes), int(nbytes) // 4
        self.s, self.engine, self.tune = float(s), engine, dict(tune or {})
        self.right = (self.rank + 1) % self.world
        self.left = (self.rank - 1) % self.world
        torch.cuda.set_device(device)
        self.pads = SignalPads(comm, device, timeout_s=timeout_s)
        self.recv = SymmetricBuffer(comm, nbytes, device)          # neighbour writes here
        dev = torch.device("cuda", device)
        self.n_total = self.n * self.compute_ratio
        self.a = torch.empty(self.n_total, dtype=torch.float32, device=dev)
        self.b = torch.empty(self.n_total, dtype=torch.float32, device=dev)
        self.c = torch.empty(self.n_total, dtype=torch.float32, device=dev)
        self.C.fill_triad_inputs(self.b.data_ptr(), self.c.data_ptr(), self.n_total, self.rank, self._stream())
        self.epoch = 0
        self.launches = 0
        self._counter = torch.zeros(1, dtype=torch.int64, device=dev)
        # e2e path: pinned host staging + a copy stream
        self._host_c: Optional[torch.Tensor] = None
        self._host_out = torch.zeros(1, dtype=torch.int64).pin_memory() if torch.cuda.is_available() else None
        self._h2d = torch.cuda.Stream(device)
        torch.cuda.synchronize(device)
        comm.barrier()

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ---- device-resident step (what `value` in bench.py times) -----------------------
    def step(self, put: bool = True) -> None:
        self.epoch += 1
        C = self.C
        sync = self.pads.sync_ops(signal_rank=self.right if put else None, signal_section=C.PAD_DONE,
                                  epoch=self.epoch)
        arrive = self.pads.word(self.rank, C.PAD_DONE + self.left) if put else 0
        ctas = C.triad_put(self.a.data_ptr(), self.recv.ptrs[self.right] if put else 0,
                           self.b.data_ptr(), self.c.data_ptr(), self.s, self.n_total, self.engine, self.tune,
                           sync, arrive, self.epoch, self.device, self._stream(), self.n)
        self.pads.advance_tickets(ctas)
        self.launches += 1

    # ---- unfused building blocks (for overlap % and the stock comparison) --------------
    def triad_only(self) -> None:
        self.C.triad_put(self.a.data_ptr(), 0, self.b.data_ptr(), self.c.data_ptr(), self.s, self.n_total,
                         self.engine, self.tune, {}, 0, 0, self.device, self._stream(), self.n)
        self.launches += 1

    def put_only(self) -> None:
        """Plain put of `a` with the K-p2p kernel (+ arrival wait), no compute."""
        self.epoch += 1
        C = self.C
        sync = self.pads.sync_ops(signal_rank=self.right, signal_section=C.PAD_DONE, epoch=self.epoch)
        ctas = C.copy(self.recv.ptrs[self.right], self.a.data_ptr(), self.nbytes, False, self.engine,
                      self.tune, sync, self.device, self._stream())
        self.pads.advance_tickets(ctas)
        C.wait(self.pads.word(self.rank, C.PAD_DONE + self.left), self.epoch, self.pads.timeout_ns,
               self.pads.status_ptr, self._stream())
        self.launches += 2

    def stock_step(self, how: str = "memcpy") -> None:
        """The reference *pattern* through stock calls: triad kernel, then a library transfer."""
        self.triad_only()
        if self.world == 1:
            self.C.memcpy_async(self.recv.ptrs[0], self.a.data_ptr(), self.nbytes, self._stream())
        elif how == "memcpy":
            # cudaMemcpyPeerAsync needs device ordinals of this process' view; peer pointers are
            # IPC mappings, so a default-kind async copy takes the same copy-engine path.
            self.C.memcpy_async(self.recv.ptrs[self.right], self.a.data_ptr(), self.nbytes, self._stream())
        elif how == "nccl":
            import torch.distributed as dist
            recv_t = self.recv.tensor(torch.float32)
            # the message is the halo: the first n elements of `a` (a holds compute_ratio * n elements)
            ops = [dist.P2POp(dist.isend, self.a[:self.n], self.right), dist.P2POp(dist.irecv, recv_t, self.left)]
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        else:
            raise ValueError(how)

    # ---- end-to-end step through host memory -------------------------------------------
    def make_host_input(self) -> torch.Tensor:
        """Pinned host copy of the halo part of this rank's `c` — the per-step input a caller hands in
        (the interior of the local domain stays resident on the device)."""
        if self._host_c is None:
            self._host_c = self.c[:self.n].cpu().pin_memory()
        return self._host_c

    def step_from_host(self, c_host: torch.Tensor, chunks: int = 8) -> int:
        """Public end-to-end step: H2D of the step's input `c` (pinned), fused triad+put,
        receiver-side check, D2H of the 8-byte result.  The H2D copy is chunked on a copy
        stream and each chunk's fused kernel starts as soon as its bytes are on the device.
        Returns the number of wrong words received from the left neighbour."""
        C = self.C
        self.epoch += 1
        n = self.n
        per = ((n + chunks - 1) // chunks + 3) // 4 * 4
        main = torch.cuda.current_stream(self.device)
        self._h2d.wait_stream(main)
        if self.compute_ratio > 1:
            # Interior of the local domain: needs nothing from the host, runs under the H2D copies.
            C.triad_put(self.a.data_ptr() + 4 * n, 0, self.b.data_ptr() + 4 * n, self.c.data_ptr() + 4 * n,
                        self.s, self.n_total - n, self.engine, self.tune, {}, 0, 0, self.device,
                        main.cuda_stream, 0)
            self.launches += 1
        off = 0
        k = 0
        while off < n:
            m = min(per, n - off)
            last = off + m >= n
            with torch.cuda.stream(self._h2d):
                self.c[off:off + m].copy_(c_host[off:off + m], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._h2d)
            main.wait_event(ev)
            sync = self.pads.sync_ops(signal_rank=self.right if last else None,
                                      signal_section=C.PAD_DONE, epoch=self.epoch)
            arrive = self.pads.word(self.rank, C.PAD_DONE + self.left) if last else 0
            ctas = C.triad_put(self.a.data_ptr() + 4 * off, self.recv.ptrs[self.right] + 4 * off,
                               self.b.data_ptr() + 4 * off, self.c.data_ptr() + 4 * off, self.s, m,
                               self.engine, self.tune, sync, arrive, self.epoch, self.device,
                               main.cuda_stream)
            self.pads.advance_tickets(ctas)
            self.launches += 1
            off += m
            k += 1
        self._counter.zero_()
        C.verify_triad(self.recv.ptrs[self.rank], n, self.left, self.s, self._counter.data_ptr(),
                       main.cuda_stream)
        self.launches += 1
        self._host_out.copy_(self._counter, non_blocking=True)
        main.synchronize()
        return int(self._host_out.item())

    @property
    def h2d_bytes_per_step(self) -> int:
        return self.nbytes

    @property
    def d2h_bytes_per_step(self) -> int:
        return 8

    # ---- checking -------------------------------------------------------------------
    def verify(self) -> int:
        """Number of wrong words in what the left neighbour put here (exact compare)."""
        self._counter.zero_()
        self.C.verify_triad(self.recv.ptrs[self.rank], self.n, self.left, self.s,
                            self._counter.data_ptr(), self._stream())
        torch.cuda.synchronize(self.device)
        return int(self._counter.item())

    def check(self) -> None:
        self.pads.check()

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        self.recv.close()
        self.pads.close()


# =====================================================================================
@dataclass
class P2PResult:
    label: str
    transport: str
    engine: str
    nbytes: int
    ranks: int
    uni_ns: float
    bi_ns: float
    mismatches: int = 0
    extra: Dict = field(default_factory=dict)

    @property
    def pairs(self) -> int:
        return self.ranks // 2

    @property
    def uni_gbps(self) -> float:
        return bandwidth_gbps(self.nbytes, self.pairs, self.uni_ns, False)

    @property
    def bi_gbps(self) -> float:
        return bandwidth_gbps(self.nbytes, self.pairs, self.bi_ns, True)

    def lines(self, with_size: bool = False) -> List[str]:
        label = self.label + (f" [{self.nbytes} B]" if with_size else "")
        return [f"{label} Unidirectional Bandwidth: {self.uni_gbps:.6g} GB/s",
                f"{label} Bidirectional Bandwidth: {self.bi_gbps:.6g} GB/s"]

    def row(self) -> Dict:
        return {"pattern": "peer2pear", "label": self.label, "transport": self.transport,
                "engine": self.engine, "ranks": self.ranks, "bytes": self.nbytes,
                "uni_us": self.uni_ns * 1e-3, "bi_us": self.bi_ns * 1e-3,
                "uni_GBps": self.uni_gbps, "bi_GBps": self.bi_gbps,
                "uni_GBps_per_pair": self.uni_gbps / max(self.pairs, 1),
                "frac_of_450GBps_per_dir": self.uni_gbps / max(self.pairs, 1) / 450.0,
                "mismatches": self.mismatches, **self.extra}


class P2PBench:
    """Pairwise GPU<->GPU bandwidth, device-timed, max over ranks, min over iterations."""

    TRANSPORTS = ("put", "get", "hybrid", "sendrecv", "memcpy", "nccl")

    def __init__(self, comm: Comm, device: int, max_bytes: int = REFERENCE_MESSAGE_BYTES,
                 transport: str = "put", engine: str = "tma", tune: Optional[dict] = None,
                 iters: int = 10, label: str = "Tile2Tile", timeout_s: float = 30.0, put_fraction: float = 0.5):
        """``hybrid``: every message is driven from BOTH ends at once — the sender puts the first ``put_fraction`` of it
        (peer stores) while the receiver gets the rest (peer loads), two kernels on two GPUs working on one direction of
        the link.  SM-issued stores and SM-issued loads can saturate at different rates below the link's;
        together they can fill what either leaves."""
        if transport not in self.TRANSPORTS:
            raise ValueError(f"transport must be one of {self.TRANSPORTS}")
        if comm.world < 2 or comm.world % 2:
            raise ValueError("peer2pear needs an even number of ranks >= 2")
        self.C = native()
        self.comm, self.device = comm, device
        self.rank, self.world = comm.rank, comm.world
        self.transport, self.engine, self.tune = transport, engine, dict(tune or {})
        self.iters, self.label = iters, label
        torch.cuda.set_device(device)
        self.pads = SignalPads(comm, device, timeout_s=timeout_s)
        self.send = SymmetricBuffer(comm, max_bytes, device)
        self.recv = SymmetricBuffer(comm, max_bytes, device)
        self.max_bytes = max_bytes
        self.epoch = 0
        self.partner = self.rank ^ 1
        self.launches = 0
        self.put_fraction = float(put_fraction)
        self._side = torch.cuda.Stream(device) if transport == "hybrid" else None

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _seed(self, rank: int) -> int:
        return (0x9E3779B9 * (rank + 1)) & 0xFFFFFFFF

    def _enqueue(self, nbytes: int, sends_to: int, recvs_from: int) -> None:
        C, pads, me, st = self.C, self.pads, self.rank, self._stream()
        ep = self.epoch
        tr = self.transport
        if tr == "nccl":
            import torch.distributed as dist
            ops = []
            if sends_to >= 0:
                ops.append(dist.P2POp(dist.isend, self.send.tensor()[:nbytes], sends_to))
            if recvs_from >= 0:
                ops.append(dist.P2POp(dist.irecv, self.recv.tensor()[:nbytes], recvs_from))
            for w in dist.batch_isend_irecv(ops):
                w.wait()
            return
        if tr == "hybrid":
            split = int(nbytes * self.put_fraction) // 16 * 16
            main = torch.cuda.current_stream(self.device)
            if sends_to >= 0 and split > 0:          # my half of the outgoing message: peer stores
                sync = pads.sync_ops(signal_rank=sends_to, signal_section=C.PAD_DONE, epoch=ep)
                pads.advance_tickets(C.copy(self.recv.ptrs[sends_to], self.send.local_ptr, split, False, self.engine,
                                            self.tune, sync, self.device, st))
                self.launches += 1
            if recvs_from >= 0 and split < nbytes:   # the other half of the incoming message: peer loads, side stream
                self._side.wait_stream(main)
                sync = pads.sync_ops(signal_rank=recvs_from, signal_section=C.PAD_ACK, epoch=ep)
                sync["ticket"] = pads.word(me, C.PAD_LOCAL + 1)          # second ticket counter: concurrent kernel
                sync["ticket_base"] = getattr(self, "_side_tickets", 0) & 0xFFFFFFFF
                ctas = C.copy(self.recv.local_ptr + split, self.send.ptrs[recvs_from] + split, nbytes - split, True,
                              self.engine, self.tune, sync, self.device, self._side.cuda_stream)
                self._side_tickets = getattr(self, "_side_tickets", 0) + ctas
                main.wait_stream(self._side)
                self.launches += 1
            if recvs_from >= 0 and split > 0:
                C.wait(pads.word(me, C.PAD_DONE + recvs_from), ep, pads.timeout_ns, pads.status_ptr, st)
                self.launches += 1
            if sends_to >= 0 and split < nbytes:     # owner: my buffer is free once the reader is done
                C.wait(pads.word(me, C.PAD_ACK + sends_to), ep, pads.timeout_ns, pads.status_ptr, st)
                self.launches += 1
            return
        if tr == "sendrecv" and recvs_from >= 0:
            C.signal(pads.word(recvs_from, C.PAD_READY + me), ep, st)
            self.launches += 1
        if sends_to >= 0 and tr != "get":
            sync = pads.sync_ops(signal_rank=sends_to, signal_section=C.PAD_DONE, epoch=ep,
                                 wait_section=C.PAD_READY if tr == "sendrecv" else None,
                                 wait_rank=sends_to)
            if tr == "memcpy":
                C.memcpy_async(self.recv.ptrs[sends_to], self.send.local_ptr, nbytes, st)
                C.signal(sync["signal_flag"], ep, st)
            else:
                pads.advance_tickets(C.copy(self.recv.ptrs[sends_to], self.send.local_ptr, nbytes, False,
                                            self.engine, self.tune, sync, self.device, st))
            self.launches += 1
        if recvs_from >= 0:
            if tr == "get":
                sync = pads.sync_ops(signal_rank=recvs_from, signal_section=C.PAD_ACK, epoch=ep)
                pads.advance_tickets(C.copy(self.recv.local_ptr, self.send.ptrs[recvs_from], nbytes, True,
                                            self.engine, self.tune, sync, self.device, st))
            else:
                C.wait(pads.word(me, C.PAD_DONE + recvs_from), ep, pads.timeout_ns, pads.status_ptr, st)
            self.launches += 1
        if tr == "get" and sends_to >= 0:
            C.wait(pads.word(me, C.PAD_ACK + sends_to), ep, pads.timeout_ns, pads.status_ptr, st)
            self.launches += 1

    def _phase(self, nbytes: int, sends_to: int, recvs_from: int) -> float:
        best = float("inf")
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        stream = torch.cuda.current_stream(self.device)
        for _ in range(self.iters):
            self.epoch += 1
            self.comm.barrier()
            self.pads.device_barrier(stream.cuda_stream)
            torch.cuda.nvtx.range_push(f"peer2pear {self.transport} {nbytes} B")
            e0.record(stream)
            self._enqueue(nbytes, sends_to, recvs_from)
            e1.record(stream)
            torch.cuda.nvtx.range_pop()
            stream.synchronize()
            self.pads.check()
            best = min(best, self.comm.max(e0.elapsed_time(e1) * 1e6))
        return best

    def run(self, nbytes: int = REFERENCE_MESSAGE_BYTES, verify: bool = True) -> P2PResult:
        if nbytes % 16 or nbytes > self.max_bytes:
            raise ValueError("bad message size")
        C, me, partner = self.C, self.rank, self.partner
        even = me % 2 == 0
        st = self._stream()
        C.fill_pattern(self.send.local_ptr, nbytes // 4, self._seed(me), st)
        C.memset_async(self.recv.local_ptr, 0, nbytes, st)
        torch.cuda.synchronize(self.device)
        self.comm.barrier()
        uni = self._phase(nbytes, partner if even else -1, -1 if even else partner)
        bad = 0
        if verify and not even:
            bad += self._verify(nbytes, partner)
        C.memset_async(self.recv.local_ptr, 0, nbytes, self._stream())
        torch.cuda.synchronize(self.device)
        self.comm.barrier()
        bi = self._phase(nbytes, partner, partner)
        if verify:
            bad += self._verify(nbytes, partner)
        bad = int(self.comm.sum(bad))
        return P2PResult(self.label, self.transport, self.engine, nbytes, self.world, uni, bi, bad)

    def _verify(self, nbytes: int, sender: int) -> int:
        counters = torch.zeros(2, dtype=torch.int64, device=torch.device("cuda", self.device))
        self.C.verify_pattern(self.recv.local_ptr, nbytes // 4, self._seed(sender), counters.data_ptr(),
                              counters.data_ptr() + 8, 0, 0, 0, 0, self._stream())
        torch.cuda.synchronize(self.device)
        return int(counters[0].item())

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        self.send.close()
        self.recv.close()
        self.pads.close()


def main(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200.models.peer2pear [label] [--sweep] ...``"""
    import argparse

    ap = argparse.ArgumentParser(prog="peer2pear")
    ap.add_argument("label", nargs="?", default="Tile2Tile")
    ap.add_argument("--transport", default="put", choices=P2PBench.TRANSPORTS)
    ap.add_argument("--engine", default="tma", choices=("ldst", "tma"))
    ap.add_argument("--bytes", type=int, action="append")
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args(argv)
    comm = Comm()
    device = comm.device   # chosen before the process group was bound to it (Comm.pick_device)
    sizes = sweep_sizes() if args.sweep else (args.bytes or [REFERENCE_MESSAGE_BYTES])
    bench = P2PBench(comm, device, max(sizes), args.transport, args.engine, iters=args.iters,
                     label=args.label)
    rc = 0
    for nbytes in sizes:
        res = bench.run(nbytes)
        if comm.rank == 0:
            for line in res.lines(with_size=len(sizes) > 1):
                print(line, flush=True)
            if res.mismatches:
                print(f"{args.label} VERIFICATION FAILED: {res.mismatches} wrong words", flush=True)
                rc = 1
            if args.json:
                with open(args.json, "a") as f:
                    f.write(json.dumps(res.row()) + "\n")
    bench.close()
    comm.close()
    return rc


if __name__ == "__main__":
    raise SystemExit(main())
