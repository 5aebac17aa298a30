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

``AlltoallvMiniapp`` / ``VirtualAlltoallv`` are the all-to-all-v with device-resident counts (``bin/alltoall
--counts``): rows of ``row_bytes``, per-peer int64 counts in peer-mapped memory, read by the kernel itself, so an
``exchange(x, splits)`` never synchronises the host.  Its ``nccl`` algorithm is the stock MoE path: an all-to-all of
the counts, ``.tolist()`` (a device-to-host sync), then ``all_to_all_single`` with split sizes.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from .. import native
from ..ops.alltoall import (all_gather, all_to_all, all_to_all_v, as_blocks, check_args, check_gather_args,
                             check_v_args, check_verdict)
from ..parallel.comm import Comm
from ..parallel.local import VirtualRanks
from ..parallel.symmetric import SignalPads, SymmetricBuffer
from .collective import CollectiveMiniapp, gbps, report

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
        return {"pattern": "alltoall", "variant": self.variant, "ranks": self.world, "block_bytes": self.block_bytes,
                "ms": self.ms, "GBps_sent_per_rank": gbps(sent, self.ms), "ctas": self.ctas,
                "mismatches": self.mismatches}


class AlltoallMiniapp(CollectiveMiniapp):
    PATTERN = "alltoall"

    def __init__(self, comm: Comm, device: int, block_bytes: int = 16 << 20, algo: str = "push", ctas: int = 0,
                 timeout_s: float = 30.0, _shared: Optional[dict] = None):
        """``_shared``: buffers made by an in-process group (``VirtualAlltoall``): ``pads``, ``send``, ``recv``."""
        if algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}")
        check_args(comm.world, block_bytes)
        super().__init__(comm, device, native(), algo, ctas, _shared, VIRTUAL_ALGOS)
        self.block_bytes = int(block_bytes)
        self.nbytes = self.world * self.block_bytes
        self.generation = 0           # iterations initialised so far: the pattern seeds of the last one are checked
        if _shared is not None:
            self.pads, self.send, self.recv = _shared["pads"], _shared["send"], _shared["recv"]
        else:
            self.pads = SignalPads(comm, device, timeout_s=timeout_s)
            self.send = SymmetricBuffer(comm, self.nbytes, device, zero=False)
            self.recv = SymmetricBuffer(comm, self.nbytes, device, zero=False)

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

    def result(self, ms: float, mismatches: int) -> AlltoallResult:
        return AlltoallResult(self.algo, self.world, self.block_bytes, ms, mismatches, self.launch_ctas)


class VirtualAlltoall(VirtualRanks):
    """``world`` AlltoallMiniapp ranks on one GPU (``VirtualRanks``)."""

    def __init__(self, world: int, block_bytes: int, algo: str = "push", ctas: int = 0, device: int = 0,
                 timeout_s: float = 10.0):
        self.refuse(world, algo, VIRTUAL_ALGOS)
        check_args(world, block_bytes)
        super().__init__(world, device, ctas)
        self.block_bytes = int(block_bytes)
        pads = self.group.pads(timeout_s=timeout_s)
        send = self.group.symmetric(world * self.block_bytes, zero=False)
        recv = self.group.symmetric(world * self.block_bytes, zero=False)
        self.ranks: List[AlltoallMiniapp] = [
            AlltoallMiniapp(self.group.comms[r], device, self.block_bytes, algo, ctas=self.ctas, timeout_s=timeout_s,
                            _shared={"pads": pads[r], "send": send[r], "recv": recv[r]})
            for r in range(world)]

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

    def results(self) -> List[torch.Tensor]:
        """The receive buffer of every rank as a [P, B] uint8 tensor on the host."""
        self.synchronize()
        return [app.recv.tensor().cpu().reshape(self.world, self.block_bytes) for app in self.ranks]


# ---------------------------------------------------------------------------------------------------- all-to-all-v ----
V_ALGOS = ("push", "pull", "nccl")
COUNT_KINDS = ("random", "skewed", "equal")
TAIL_POISON_SEED = 0xC0DE0001
_M64 = (1 << 64) - 1


def _mix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def mean_rows(block_bytes: int, row_bytes: int) -> int:
    """--block-bytes as the mean segment, rounded to rows (at least one)."""
    return max(1, (block_bytes + row_bytes // 2) // row_bytes)


def draw_counts(kind: str, world: int, mean: int, it: int) -> List[List[int]]:
    """The count matrix of iteration ``it`` (M[p][q] rows from p to q), as bin/alltoall --counts draws it: ``random``
    0 ... 2*mean per pair and one pair 0; ``skewed`` 2*mean into the hot rank it % P and at most mean/P into the others;
    ``equal`` the mean for every pair.
    Every matrix fits capacities of 2*P*mean rows."""
    if kind not in COUNT_KINDS:
        raise ValueError(f"--counts must be random, skewed or equal, not {kind}")
    hot = it % world
    m = [[0] * world for _ in range(world)]
    for p in range(world):
        for q in range(world):
            h = _mix64((it << 16) | (p << 8) | q)
            m[p][q] = (mean if kind == "equal" else (2 * mean if q == hot else h % (mean // world + 1))
                       if kind == "skewed" else h % (2 * mean + 1))
    if kind == "random":
        i = _mix64(0xA11 ^ (it << 32)) % (world * world)
        m[i // world][i % world] = 0
    return m


@dataclass
class AlltoallvResult:
    variant: str
    world: int
    block_bytes: int
    row_bytes: int
    counts: str
    ms: float
    mismatches: int
    off_rank_bytes: float
    max_bytes_into_a_rank: float
    ctas: int = 0

    def row(self) -> dict:
        """One JSON row with the CLI's keys; GB/s is off-rank bytes summed over ranks / P / time."""
        return {"pattern": "alltoallv", "variant": self.variant, "ranks": self.world, "block_bytes": self.block_bytes,
                "ms": self.ms, "GBps_sent_per_rank": gbps(self.off_rank_bytes / self.world, self.ms),
                "ctas": self.ctas, "mismatches": self.mismatches,
                "counts": self.counts, "row_bytes": self.row_bytes,
                "max_bytes_into_a_rank": self.max_bytes_into_a_rank}


class AlltoallvMiniapp(CollectiveMiniapp):
    """One rank of the all-to-all-v.  ``capacity_rows`` rows of ``row_bytes`` are allocated for the send and for the
    receive buffer and declared to the kernel (``send_capacity_rows`` / ``recv_capacity_rows``; they must be the same
    on every rank).  ``exchange(x, splits)`` is the enqueue-only entry point; ``run()`` is the CLI's timed, checked loop."""

    PATTERN = "alltoallv"
    BUFFERS = ("send", "recv", "counts")

    def __init__(self, comm: Comm, device: int, row_bytes: int, capacity_rows: int, algo: str = "push", ctas: int = 0,
                 timeout_s: float = 30.0, _shared: Optional[dict] = None):
        """``_shared``: buffers made by an in-process group (``VirtualAlltoallv``): ``pads``, ``send``, ``recv``,
        ``counts``."""
        if algo not in V_ALGOS:
            raise ValueError(f"algo must be one of {V_ALGOS}")
        check_v_args(comm.world, row_bytes, capacity_rows, capacity_rows)
        super().__init__(comm, device, native(), algo, ctas, _shared, VIRTUAL_ALGOS)
        self.row_bytes = int(row_bytes)
        self.send_capacity_rows = self.recv_capacity_rows = int(capacity_rows)
        self.nbytes = int(capacity_rows) * self.row_bytes
        self.generation = 0
        self.matrix: List[List[int]] = []       # run(): the count matrix of the last initialised iteration
        if _shared is not None:
            self.pads, self.send, self.recv = _shared["pads"], _shared["send"], _shared["recv"]
            self.counts = _shared["counts"]
        else:
            self.pads = SignalPads(comm, device, timeout_s=timeout_s)
            self.send = SymmetricBuffer(comm, self.nbytes, device, zero=False)
            self.recv = SymmetricBuffer(comm, self.nbytes, device, zero=False)
            self.counts = SymmetricBuffer(comm, 8 * self.world, device, zero=True)
        dev = torch.device("cuda", device)
        self.recv_counts = torch.zeros(self.world, dtype=torch.int64, device=dev)
        self.verdict_word = torch.zeros(1, dtype=torch.int32, device=dev)

    def rows(self, buf: SymmetricBuffer, dtype: torch.dtype = torch.uint8) -> torch.Tensor:
        """``buf`` (send or recv) as [capacity_rows, row] of ``dtype``."""
        return buf.tensor(dtype).view(self.nbytes // self.row_bytes, -1)

    def run_once(self) -> None:
        """Enqueue one all-to-all-v of what the send and counts buffers hold.  Precondition: every rank's send buffer
        and counts are final and no rank still reads its receive buffer or recv_counts (``run()`` and ``exchange()``
        put ``pads.device_barrier`` before it)."""
        pads, st = self.pads, self._stream()
        if self.algo == "nccl":
            self._run_nccl()
            return
        pads.barrier_epoch += 1
        self.launch_ctas = all_to_all_v(self.send.ptrs, self.recv.ptrs, self.counts.ptrs, self.recv_counts.data_ptr(),
                                        self.verdict_word.data_ptr(), pads.buf.ptrs, pads.ticket_ptr,
                                        pads.ticket_issued, self.rank, self.row_bytes, self.send_capacity_rows,
                                        self.recv_capacity_rows, pads.barrier_epoch, pads.timeout_ns, pads.status_ptr,
                                        self.ctas, self.device, st, self.algo == "pull")
        pads.advance_tickets(self.launch_ctas)

    def _run_nccl(self) -> None:
        """The stock path: counts all-to-all, .tolist() (the host sync), all_to_all_single with split sizes."""
        import torch.distributed as dist

        send_counts = self.counts.tensor(torch.int64)
        if self.world > 1:
            dist.all_to_all_single(self.recv_counts, send_counts)
        else:
            self.recv_counts.copy_(send_counts)
        ins, outs = send_counts.tolist(), self.recv_counts.tolist()
        if min(ins + outs) < 0 or sum(ins) > self.send_capacity_rows or sum(outs) > self.recv_capacity_rows:
            raise ValueError("all-to-all-v: the counts do not fit the capacities")
        rb = self.row_bytes
        src, dst = self.send.tensor()[: sum(ins) * rb], self.recv.tensor()[: sum(outs) * rb]
        if self.world > 1:
            dist.all_to_all_single(dst, src, [c * rb for c in outs], [c * rb for c in ins])
        else:
            dst.copy_(src)

    def exchange(self, x: torch.Tensor, splits: torch.Tensor):
        """Send the rows of ``x`` ([n, row_bytes worth of any dtype], n <= capacity) split by ``splits`` (device
        int64[P]: rows for every rank, in rank order).  Enqueues the copies into the symmetric buffers, the device
        barrier and the launch on the current stream and returns (received rows as [capacity, row] of x's dtype,
        recv_counts); rows past sum(recv_counts) are not written.  Never synchronises the host; a refused count matrix
        raises at ``check()``."""
        if x.shape[0] > self.send_capacity_rows:
            raise ValueError(f"all-to-all-v: x has {x.shape[0]} rows, the send capacity is {self.send_capacity_rows}")
        xb = x.contiguous().view(torch.uint8).reshape(x.shape[0], -1)
        if xb.shape[1] != self.row_bytes:
            raise ValueError(f"all-to-all-v: a row of x must hold {self.row_bytes} bytes")
        self.rows(self.send)[: x.shape[0]].copy_(xb)
        self.counts.tensor(torch.int64).copy_(splits)
        self.pads.device_barrier(self._stream())
        self.run_once()
        return self.rows(self.recv, x.dtype), self.recv_counts

    def verdict(self) -> int:
        """The verdict word of the last launch (synchronises)."""
        torch.cuda.synchronize(self.device)
        return int(self.verdict_word.item())

    def check(self) -> None:
        """Synchronise; RuntimeError on a failed device-side wait, ValueError with the verdict's words on a refused
        count matrix."""
        torch.cuda.synchronize(self.device)
        self.pads.check()
        if self.algo != "nccl":
            check_verdict(self.verdict())

    # ---- the CLI's seeded loop --------------------------------------------------------------------------------
    def initialize(self, kind: str, mean: int) -> None:
        """A new iteration: draw the count matrix, my send segments <- the pattern of (rank, q) at their packed rows,
        the receive buffer <- the poison (past my total: the tail poison), my counts <- my row of the matrix."""
        P, rb, st = self.world, self.row_bytes, self._stream()
        m = self.matrix = draw_counts(kind, P, mean, self.generation)
        total = sum(m[p][self.rank] for p in range(P))
        cap = self.nbytes // rb
        self.C.fill_pattern(self.recv.local_ptr + total * rb, (cap - total) * rb // 4, TAIL_POISON_SEED, st)
        off = 0
        for q in range(P):
            self.C.fill_pattern(self.send.local_ptr + off * rb, m[self.rank][q] * rb // 4,
                                pair_seed(self.generation, self.rank, q), st)
            off += m[self.rank][q]
        self.C.fill_pattern(self.recv.local_ptr, total * rb // 4, POISON_SEED, st)
        self.counts.tensor(torch.int64).copy_(torch.tensor(m[self.rank], dtype=torch.int64))
        self.recv_counts.fill_(-1)
        self.generation += 1

    def mismatches(self) -> int:
        """Wrong words of the receive buffer against the last iteration (segment from p at its packed row, the tail
        poison past the total), plus one per wrong recv_count and one for a non-zero verdict (kernels only)."""
        P, rb, st, m = self.world, self.row_bytes, self._stream(), self.matrix
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        off = 0
        for p in range(P):
            self.C.verify_pattern(self.recv.local_ptr + off * rb, m[p][self.rank] * rb // 4,
                                  pair_seed(self.generation - 1, p, self.rank), count.data_ptr(), stream=st)
            off += m[p][self.rank]
        self.C.verify_pattern(self.recv.local_ptr + off * rb, (self.nbytes // rb - off) * rb // 4, TAIL_POISON_SEED,
                              count.data_ptr(), stream=st)
        torch.cuda.synchronize(self.device)
        bad = int(count.item())
        bad += sum(int(a != b) for a, b in zip(self.recv_counts.tolist(), [m[p][self.rank] for p in range(P)]))
        if self.algo != "nccl":
            bad += int(int(self.verdict_word.item()) != 0)
        return bad

    def run(self, kind: str, block_bytes: int, iters: int = 5, warmup: int = 1) -> AlltoallvResult:
        """``iters`` timed all-to-all-v's of freshly drawn counts with mean segments of ``block_bytes`` (rounded to
        rows); capacity_rows must be at least 2 * P * mean."""
        mean = mean_rows(block_bytes, self.row_bytes)
        if 2 * self.world * mean > self.send_capacity_rows:
            raise ValueError(f"all-to-all-v: --counts needs {2 * self.world * mean} rows of capacity")
        self._kind, self._block_bytes, self._traffic = kind, block_bytes, (0.0, 0.0)
        return super().run(iters, warmup, kind, mean)

    def at_best(self) -> None:
        self._traffic = _traffic(self.matrix, self.row_bytes)

    def result(self, ms: float, mismatches: int) -> AlltoallvResult:
        return AlltoallvResult(self.algo, self.world, self._block_bytes, self.row_bytes, self._kind, ms, mismatches,
                               *self._traffic, ctas=self.launch_ctas)


def _traffic(m: List[List[int]], row_bytes: int):
    """(off-rank bytes of all ranks, the most bytes any rank receives)."""
    P = len(m)
    off = sum(m[p][q] for p in range(P) for q in range(P) if p != q) * row_bytes
    into = max(sum(m[p][q] for p in range(P)) for q in range(P)) * row_bytes
    return float(off), float(into)


class VirtualAlltoallv(VirtualRanks):
    """``world`` AlltoallvMiniapp ranks on one GPU (``VirtualRanks``)."""

    def __init__(self, world: int, row_bytes: int, capacity_rows: int, algo: str = "push", ctas: int = 0,
                 device: int = 0, timeout_s: float = 10.0):
        self.refuse(world, algo, VIRTUAL_ALGOS)
        check_v_args(world, row_bytes, capacity_rows, capacity_rows)
        super().__init__(world, device, ctas)
        self.row_bytes, self.capacity_rows = int(row_bytes), int(capacity_rows)
        pads = self.group.pads(timeout_s=timeout_s)
        send = self.group.symmetric(self.capacity_rows * self.row_bytes, zero=False)
        recv = self.group.symmetric(self.capacity_rows * self.row_bytes, zero=False)
        counts = self.group.symmetric(8 * world, zero=True)
        self.ranks: List[AlltoallvMiniapp] = [
            AlltoallvMiniapp(self.group.comms[r], device, self.row_bytes, self.capacity_rows, algo, ctas=self.ctas,
                             timeout_s=timeout_s,
                             _shared={"pads": pads[r], "send": send[r], "recv": recv[r], "counts": counts[r]})
            for r in range(world)]

    def load(self, sends: List[torch.Tensor], counts: List) -> None:
        """Rank r's send buffer <- ``sends[r]`` (rows of row_bytes, any dtype, at most capacity_rows) and its counts
        <- ``counts[r]`` (P int64 values: rows for every rank).  The counts are not judged here: the kernel does."""
        if len(sends) != self.world or len(counts) != self.world:
            raise ValueError(f"one send tensor and one count row per rank ({self.world})")
        torch.cuda.synchronize(self.device)
        for app, s, c in zip(self.ranks, sends, counts):
            b = s.contiguous().view(torch.uint8).reshape(-1)
            if b.numel() > app.nbytes or b.numel() % self.row_bytes:
                raise ValueError(f"a send tensor must hold whole rows of {self.row_bytes} bytes, at most "
                                 f"{self.capacity_rows}")
            app.send.tensor()[: b.numel()].copy_(b)
            app.counts.tensor(torch.int64).copy_(torch.as_tensor(c, dtype=torch.int64).reshape(self.world))
        torch.cuda.synchronize(self.device)

    def verdicts(self) -> List[int]:
        """Every rank's verdict word of the last launch."""
        self.synchronize()
        return [int(app.verdict_word.item()) for app in self.ranks]

    def results(self):
        """Every rank's (received rows trimmed to its total as [total, row_bytes] uint8, recv_counts) on the host;
        ValueError with the words of a refused count matrix."""
        for v in self.verdicts():
            check_verdict(v)
        out = []
        for app in self.ranks:
            rc = app.recv_counts.cpu()
            total = int(rc.sum())
            out.append((app.rows(app.recv)[:total].cpu(), rc))
        return out


# ------------------------------------------------------------------------------------------------------ all-gather ----
# ``AllgatherMiniapp`` is the Python twin of ``bin/allgather`` (↔ MPI_Allgather, ncclAllGather): every rank holds one
# send block of ``block_bytes``; afterwards block p of every rank's receive buffer is rank p's block
# (``ops.alltoall.all_gather``).  Algorithms: ``push`` (default), ``pull`` and ``nccl``
# (torch.distributed.all_gather_into_tensor, the baseline).  The check is the all-to-all's: rank p's block holds the
# pattern seed of (p, iteration), the receive buffer the poison, and every block p is verified at its slot.


def gather_seed(it: int, src: int) -> int:
    """The pattern seed of rank ``src``'s send block in iteration ``it`` (never the poison)."""
    return 0x20000000 | ((it & 0x3FFFFF) << 4) | src


@dataclass
class AllgatherResult(AlltoallResult):
    def row(self) -> dict:
        row = super().row()
        row["pattern"] = "allgather"
        return row


class AllgatherMiniapp(CollectiveMiniapp):
    PATTERN = "allgather"

    def __init__(self, comm: Comm, device: int, block_bytes: int = 16 << 20, algo: str = "push", ctas: int = 0,
                 timeout_s: float = 30.0, _shared: Optional[dict] = None):
        """``_shared``: buffers made by an in-process group (``VirtualAllgather``): ``pads``, ``send``, ``recv``."""
        if algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}")
        check_gather_args(comm.world, block_bytes)
        super().__init__(comm, device, native(), algo, ctas, _shared, VIRTUAL_ALGOS)
        self.block_bytes = int(block_bytes)
        self.nbytes = self.world * self.block_bytes
        self.generation = 0
        if _shared is not None:
            self.pads, self.send, self.recv = _shared["pads"], _shared["send"], _shared["recv"]
        else:
            self.pads = SignalPads(comm, device, timeout_s=timeout_s)
            self.send = SymmetricBuffer(comm, self.block_bytes, device, zero=False)
            self.recv = SymmetricBuffer(comm, self.nbytes, device, zero=False)

    def initialize(self) -> None:
        """My send block <- the pattern of (rank, a new iteration); the receive buffer <- the poison."""
        st = self._stream()
        self.C.fill_pattern(self.send.local_ptr, self.block_bytes // 4, gather_seed(self.generation, self.rank), st)
        self.C.fill_pattern(self.recv.local_ptr, self.nbytes // 4, POISON_SEED, st)
        self.generation += 1

    def run_once(self) -> None:
        """Enqueue one all-gather on the current stream (precondition as ``AlltoallMiniapp.run_once``)."""
        pads, st = self.pads, self._stream()
        if self.algo == "nccl":
            import torch.distributed as dist
            src, dst = self.send.tensor(), self.recv.tensor()
            if self.world > 1:
                dist.all_gather_into_tensor(dst, src)
            else:
                dst.copy_(src)
            return
        pads.barrier_epoch += 1
        self.launch_ctas = all_gather(self.send.ptrs, self.recv.ptrs, pads.buf.ptrs, pads.ticket_ptr,
                                      pads.ticket_issued, self.rank, self.block_bytes, pads.barrier_epoch,
                                      pads.timeout_ns, pads.status_ptr, self.ctas, self.device, st,
                                      self.algo == "pull")
        pads.advance_tickets(self.launch_ctas)

    def all_gather(self, x: torch.Tensor) -> torch.Tensor:
        """All-gather the tensor ``x`` (``block_bytes`` of any dtype): copy it into the symmetric send block, the device
        barrier and the launch, all enqueued on the current stream; returns the receive buffer as a [P, *x.shape] view
        of x's dtype, which the next call overwrites.  Never synchronises the host."""
        xb = x.contiguous().view(torch.uint8).reshape(-1)
        if xb.numel() != self.block_bytes:
            raise ValueError(f"all-gather: x must hold {self.block_bytes} bytes")
        self.send.tensor().copy_(xb)
        if self.algo != "nccl":
            self.pads.device_barrier(self._stream())
        self.run_once()
        return self.recv.tensor().view(x.dtype).reshape(self.world, *x.shape)

    def mismatches(self) -> int:
        """Wrong words of the receive buffer (block p must be rank p's) and of my send block (it must be unchanged)."""
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        st, B, it = self._stream(), self.block_bytes, self.generation - 1
        for p in range(self.world):
            self.C.verify_pattern(self.recv.local_ptr + p * B, B // 4, gather_seed(it, p), count.data_ptr(),
                                  stream=st)
        self.C.verify_pattern(self.send.local_ptr, B // 4, gather_seed(it, self.rank), count.data_ptr(), stream=st)
        torch.cuda.synchronize(self.device)
        return int(count.item())

    def result(self, ms: float, mismatches: int) -> AllgatherResult:
        return AllgatherResult(self.algo, self.world, self.block_bytes, ms, mismatches, self.launch_ctas)


class VirtualAllgather(VirtualRanks):
    """``world`` AllgatherMiniapp ranks on one GPU (``VirtualRanks``)."""

    def __init__(self, world: int, block_bytes: int, algo: str = "push", ctas: int = 0, device: int = 0,
                 timeout_s: float = 10.0):
        self.refuse(world, algo, VIRTUAL_ALGOS)
        check_gather_args(world, block_bytes)
        super().__init__(world, device, ctas)
        self.block_bytes = int(block_bytes)
        pads = self.group.pads(timeout_s=timeout_s)
        send = self.group.symmetric(self.block_bytes, zero=False)
        recv = self.group.symmetric(world * self.block_bytes, zero=False)
        self.ranks: List[AllgatherMiniapp] = [
            AllgatherMiniapp(self.group.comms[r], device, self.block_bytes, algo, ctas=self.ctas, timeout_s=timeout_s,
                             _shared={"pads": pads[r], "send": send[r], "recv": recv[r]})
            for r in range(world)]

    def load(self, sends: List[torch.Tensor]) -> None:
        """Send block of rank r <- the bytes of ``sends[r]`` (``block_bytes`` of any dtype)."""
        if len(sends) != self.world:
            raise ValueError(f"one send tensor per rank ({self.world})")
        torch.cuda.synchronize(self.device)
        for app, s in zip(self.ranks, sends):
            b = s.contiguous().view(torch.uint8).reshape(-1)
            if b.numel() != self.block_bytes:
                raise ValueError(f"a send tensor must hold {self.block_bytes} bytes")
            app.send.tensor().copy_(b)
        torch.cuda.synchronize(self.device)

    def results(self) -> List[torch.Tensor]:
        """The receive buffer of every rank as a [P, B] uint8 tensor on the host."""
        self.synchronize()
        return [app.recv.tensor().cpu().reshape(self.world, self.block_bytes) for app in self.ranks]


def main_allgather(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200 allgather [--block-bytes B] [--algo push|pull|nccl]``"""
    import argparse

    ap = argparse.ArgumentParser(prog="allgather", add_help=True)
    ap.add_argument("--block-bytes", type=int, default=16 << 20, help="bytes per rank's block (default 16 MiB)")
    ap.add_argument("--algo", default="push", choices=ALGOS)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ctas", type=int, default=0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args(argv)
    check_gather_args(1, args.block_bytes)
    comm = Comm()
    app = AllgatherMiniapp(comm, comm.device, args.block_bytes, args.algo, ctas=args.ctas)
    res = app.run(args.iters, args.warmup)
    return report(comm, app, res, args, f"allgather {args.algo} P={comm.world} B={args.block_bytes}")


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
    ap.add_argument("--counts", default=None, choices=COUNT_KINDS,
                    help="all-to-all-v with device-resident counts; --block-bytes is the mean segment")
    ap.add_argument("--row-bytes", type=int, default=16, help="with --counts: bytes per row (default 16)")
    args = ap.parse_args(argv)
    comm = Comm()
    if args.counts:
        mean = mean_rows(args.block_bytes, args.row_bytes)
        app = AlltoallvMiniapp(comm, comm.device, args.row_bytes, 2 * comm.world * mean, args.algo, ctas=args.ctas)
        res = app.run(args.counts, args.block_bytes, args.iters, args.warmup)
        what = f"alltoallv {args.algo} {args.counts} P={comm.world} B={args.block_bytes} R={args.row_bytes}"
    else:
        app = AlltoallMiniapp(comm, comm.device, args.block_bytes, args.algo, ctas=args.ctas)
        res = app.run(args.iters, args.warmup)
        what = f"alltoall {args.algo} P={comm.world} B={args.block_bytes}"
    return report(comm, app, res, args, what)


if __name__ == "__main__":
    raise SystemExit(main())
