"""Allreduce miniapp for one-process-per-GPU runs (torchrun).

Capability parity with the reference miniapps
(aurora.mpich.miniapps/src/allreduce/mpi-sycl/allreduce-mpi-sycl.cpp:88-215 and the two
OpenMP variants): every rank holds VA = rank, VC = 0; after the allreduce every
element of VC equals P(P-1)/2.  Algorithms:

  ring          fused K-ring kernel: P-1 neighbour exchanges + P accumulations, one launch
  ring-rsag     bandwidth-optimal ring, one launch: reduce-scatter + all-gather between neighbours only,
                2(P-1)/P of the block sent per rank
  ring-unfused  the reference's step structure with separate kernels (rendezvous put, then
                accumulate), no host sync between steps
  twoshot       one-launch collective over peer mappings            (↔ MPI_Allreduce, -a)
  nvls          multimem.ld_reduce / multimem.st through torch symmetric memory's multicast
  nccl          torch.distributed.all_reduce — the stock baseline
  ring-nccl     the reference pattern verbatim through stock calls: accumulate kernel,
                NCCL send/recv, host wait, P-1 times — the baseline K-ring must beat

Reductions (``op``, ↔ MPI_SUM / MPI_PROD / MPI_MIN / MPI_MAX): ``sum`` (default) accumulates into VC; ``prod``, ``min``
and ``max`` overwrite it, on every algorithm but nvls (sum-only).  Each op has its own constant-data check: max (rank r
holds r) -> P-1, min (P-r) -> 1, prod (2 on the odd ranks below 8, else 1) -> 2^min(P/2, 4).
On the integer types only (↔ MPI_BAND / MPI_BOR / MPI_BXOR / MPI_LAND / MPI_LOR / MPI_LXOR): ``band``, ``bor``,
``bxor`` act on the element bits; ``land``, ``lor``, ``lxor`` take an element as true iff it is nonzero and give 0 or 1
(at one rank VC is VA).  A floating type is refused, as MPI does, and so is ``nccl``, which has no such reductions.
Their checks are listed in ``op_input`` and ``expected_value``.
On the value-index pair types only (``float_int``, ``double_int``, ``long_int``, ``2int``, ``short_int``, ↔ MPI_FLOAT_INT
...): ``maxloc`` and ``minloc`` (↔ MPI_MAXLOC / MPI_MINLOC); the pair types take no other op.  The larger / smaller value
wins, a NaN value wins in both, -0 < +0, ties take the smaller signed index, and a combined pair's padding is zero.
``nccl`` has no such reductions and refuses them; ``ring-nccl`` moves the bytes and combines them in torch.  Their
check is ``loc_input`` / ``loc_expected`` (exact bytes).

The native single-process CLI twin is ``bin/allreduce`` (csrc/miniapps/allreduce.cu).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from .. import native
from ..ops.allreduce import (LOC_LAYOUT, check_reduce_scatter_args, loc_combine, pack_loc,
                             reduce_scatter, unpack_loc)
from ..parallel.comm import Comm
from ..parallel.local import VirtualRanks
from ..parallel.symmetric import SignalPads, SymmetricBuffer
from .collective import CollectiveMiniapp, gbps, report

ALGOS = ("ring", "ring-unfused", "twoshot", "nvls", "nccl", "ring-nccl", "ring-rsag")
VIRTUAL_ALGOS = ("ring", "ring-unfused", "twoshot", "ring-rsag")   # the ones whose peers are plain pointers (no NCCL, no multicast)
# element types of the reference's datatype trait (mpi_datatype.hpp:28-51) -> the torch dtype whose add is bit-identical
# (unsigned integers share the two's-complement add of the signed type of the same width; NCCL rows only)
# bfloat16 / half (MPICH's MPIX_C_BF16 / MPIX_C_FLOAT16): the rings round every add to the 16-bit format, two-shot sums in
# fp32 and rounds once (docs/allreduce.md)
_TORCH_DTYPE = {"float": torch.float32, "int": torch.int32, "uint": torch.int32, "double": torch.float64,
                "long": torch.int64, "ulong": torch.int64, "short": torch.int16, "ushort": torch.int16,
                "uchar": torch.uint8, "bfloat16": torch.bfloat16, "half": torch.float16}
FLOAT16_TYPES = ("bfloat16", "half")
INTEGER_OPS = ("band", "bor", "bxor", "land", "lor", "lxor")   # integer types only, as in MPI
OPS = ("sum", "prod", "min", "max") + INTEGER_OPS
_OP_ALIASES = {"product": "prod"}
UNSIGNED_TYPES = ("uint", "ulong", "ushort")   # torch stand-ins are signed: NCCL min/max would compare them signed
FLOAT_TYPES = ("float", "double") + FLOAT16_TYPES
PAIR_TYPES = tuple(LOC_LAYOUT)        # value-index pairs: maxloc / minloc only
LOC_OPS = ("maxloc", "minloc")
OPS = OPS + LOC_OPS
DTYPES = tuple(_TORCH_DTYPE) + PAIR_TYPES


def reduce_op(op: str) -> str:
    """The canonical name of a reduction (``product`` is ``prod``); ValueError if unknown."""
    op = _OP_ALIASES.get(op, op)
    if op not in OPS:
        raise ValueError(f"op must be one of {OPS} (or 'product'), not {op!r}")
    return op


def check_op_type(op: str, dtype: str) -> None:
    """ValueError if ``op`` does not reduce ``dtype``: the bitwise and logical ops take integer types only, maxloc and
    minloc the pair types only, and the pair types no other op.  The words are the native layers'."""
    op = reduce_op(op)
    if dtype in PAIR_TYPES and op not in LOC_OPS:
        raise ValueError(f"op must be maxloc or minloc for {dtype}: {op} reduces arithmetic types only")
    if op in LOC_OPS and dtype not in PAIR_TYPES:
        ops = "sum, prod, min or max" if dtype in FLOAT_TYPES else "sum, prod, min, max, band, bor, bxor, land, lor or lxor"
        raise ValueError(f"op must be {ops} for {dtype}: {op} reduces value-index pair types only")
    if op in INTEGER_OPS and dtype in FLOAT_TYPES:
        raise ValueError(f"op must be sum, prod, min or max for {dtype}: {op} reduces integer types only")


def expected_value(world: int, op: str = "sum") -> float:
    """Every element of VC after the constant-data run of ``op`` (see ``op_input``)."""
    if op == "max":
        return world - 1.0
    if op == "min":
        return 1.0
    if op == "prod":
        return 2.0 ** min(world // 2, 4)
    if op == "band":
        return 256.0 - 2 ** min(world, 4)
    if op == "bor":
        return 2.0 ** min(world, 4) - 1
    if op == "bxor":
        x = 128
        for r in range(1, world):
            x ^= r
        return float(x)
    if op == "land":
        return 1.0
    if op == "lor":
        return 1.0 if world >= 2 else 0.0
    if op == "lxor":
        return 1.0 if world >= 2 else 3.0     # one rank: VC is VA, unnormalised
    return world * (world - 1) / 2.0


def op_input(op: str, rank: int, world: int) -> float:
    """What ``rank`` holds in the constant-data run of ``op`` (exact in every type up to 16 ranks).  The integer-only
    ops' values fit in uchar, and each bitwise op's result differs from its logical twin's from 2 ranks on."""
    if op == "min":
        return float(world - rank)
    if op == "prod":
        return 2.0 if rank % 2 == 1 and rank < 8 else 1.0
    if op == "band":
        return 255.0 - 2 ** (rank % 4)
    if op == "bor":
        return 2.0 ** (rank % 4)
    if op == "bxor":
        return 128.0 if rank == 0 else float(rank)
    if op == "land":
        return rank + 1.0
    if op == "lor":
        return 2.0 * (rank % 2)
    if op == "lxor":
        return 3.0 if rank == 0 else 0.0
    return float(rank)


def vc_init(op: str, world: int) -> float:
    """VC before the constant-data run: 0 for the sum, which accumulates into it; for the other ops a value that would
    change the result if a kernel read VC instead of overwriting it."""
    return {"max": float(world), "bor": 16.0, "bxor": 64.0, "lor": 3.0, "lxor": 5.0}.get(op, 0.0)


def loc_input(op: str, rank: int, world: int):
    """(value, index) ``rank`` holds in the constant-data run of maxloc / minloc.  The result's index -1 is held by rank
    1 only, next to larger indices with the same value and a smaller index (rank 0's) with the losing value: a tie
    broken towards the larger index, an unsigned index compare and a selection by index alone each give another pair."""
    mx = op == "maxloc"
    if rank == 0:
        return (0.0 if mx else 1.0), -world - 10
    return (1.0 if mx else 0.0), 2 * rank - 3


def loc_expected(op: str, world: int):
    """(value, index) of every element of VC after the constant-data run (VC is VA at one rank)."""
    return loc_input(op, 0, 1) if world == 1 else ((1.0 if op == "maxloc" else 0.0), -1)


def loc_vc_init(op: str):
    """VC before the constant-data run: a pair that would win if a kernel read VC."""
    return (7.0 if op == "maxloc" else -7.0), -1000


def _nccl_op(op: str):
    import torch.distributed as dist
    return {"sum": dist.ReduceOp.SUM, "prod": dist.ReduceOp.PRODUCT, "min": dist.ReduceOp.MIN,
            "max": dist.ReduceOp.MAX}[op]


def bytes_sent_per_rank(algo: str, nbytes: int, world: int) -> float:
    """Faithful ring forwards the full block P-1 times; bandwidth-optimal collectives (P-1)/P of it; the ring
    reduce-scatter + all-gather (P-1)/P of it per half."""
    if algo in ("ring", "ring-unfused", "ring-nccl"):
        return float(nbytes) * (world - 1)
    if algo == "ring-rsag":
        return 2.0 * nbytes * (world - 1) / max(world, 1)
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
    op: str = "sum"

    def row(self) -> dict:
        """One JSON row; ``"op"`` only when it is not the sum (sum rows keep their shape)."""
        rate = gbps(bytes_sent_per_rank(self.algo, self.elements * self.elem_bytes, self.world), self.ms)
        row = {"pattern": "allreduce", "algo": self.algo, "type": self.dtype, "ranks": self.world,
               "elements": self.elements, "ms": self.ms, "GBps_sent_per_rank": rate,
               "frac_of_450GBps": rate / 450.0, "mismatches": self.mismatches}
        if self.op != "sum":
            row["op"] = self.op
        return row


def element_count(elem_bytes: int, world: int, log2_elems: int = 25, n_elems: int = 0) -> int:
    """Elements per rank: ``n_elems`` when given (it must split into 16-byte vectors, one slice per rank), else
    2^log2_elems rounded up to such a multiple."""
    unit = 16 // elem_bytes * world
    if n_elems:
        if n_elems < 0 or n_elems % unit:
            raise ValueError(f"n_elems must be a positive multiple of {unit} (16-byte vectors x {world} ranks)")
        return int(n_elems)
    n = 1 << log2_elems
    return -(-n // unit) * unit


def ring_layout(nbytes: int, n_chunks: int, world: int, slots_policy: int):
    """(words after the fixed signal pad, bytes of receive slots) of the fused ring: one arrival word per chunk, then
    with two slots one ack word per chunk; two blocks of slots with acks, else world-1 blocks."""
    two = slots_policy == 2
    return n_chunks * (2 if two else 1), nbytes * (2 if two else max(world - 1, 1))


def rsag_layout(nbytes: int, n_chunks: int, world: int):
    """(words after the fixed signal pad, bytes of receive slots) of the reduce-scatter + all-gather ring: one arrival
    word per chunk of a segment, world-1 segments of slots (one segment at world 1, where none is used)."""
    return n_chunks, nbytes // world * max(world - 1, 1)


def _layout(algo: str, C, n: int, esz: int, world: int, chunk_elems: int, slots_policy: int):
    """(chunks that carry an arrival word, pad words, slot bytes) of ``algo``."""
    if algo == "ring-rsag":
        n_chunks = C.ring_num_chunks(n // world, chunk_elems, esz)
        return (n_chunks,) + rsag_layout(n * esz, n_chunks, world)
    n_chunks = C.ring_num_chunks(n, chunk_elems, esz)
    return (n_chunks,) + ring_layout(n * esz, n_chunks, world, slots_policy)


class AllreduceMiniapp(CollectiveMiniapp):
    PATTERN, UNIT = "allreduce", "elements"
    BUFFERS = ("va", "vb", "vc", "slots")

    def __init__(self, comm: Comm, device: int, log2_elems: int = 25, dtype: str = "float",
                 algo: str = "ring", chunk_elems: int = 0, ctas: int = 0, timeout_s: float = 30.0,
                 slots: int = 0, pull: bool = False, n_elems: int = 0, op: str = "sum",
                 _shared: Optional[dict] = None):
        """``slots=2`` (fused ring only): two receive slots + per-chunk acks — the reference's VA/VB double
        buffer — instead of ``world-1`` slots without flow control.  ``pull=True`` (fused ring only): receiver-driven,
        every block is loaded from the left neighbour's memory instead of being stored into the right neighbour's.
        ``n_elems``: exact element count per rank instead of 2^log2_elems.  ``_shared``: buffers made by an
        in-process group (``VirtualAllreduce``): ``pads``, ``va``, ``vc`` and, where the algorithm uses them, ``vb`` and
        ``slots``.  ``op``: sum (default), prod / product, min or max; on integer types also band, bor, bxor, land, lor
        or lxor.  nvls is sum-only, nccl has no bitwise or logical reductions, and the NCCL algorithms refuse min / max
        on unsigned types (their torch stand-ins are signed)."""
        if algo not in ALGOS:
            raise ValueError(f"algo must be one of {ALGOS}")
        if dtype not in DTYPES:
            raise ValueError(f"dtype must be one of {sorted(DTYPES)}")
        op = reduce_op(op)
        check_op_type(op, dtype)
        if op != "sum" and algo == "nvls":
            raise ValueError(f"nvls reduces sums only: op={op} needs twoshot or a ring")
        if op in INTEGER_OPS and algo == "nccl":
            raise ValueError(f"nccl has no bitwise or logical reductions: op={op} needs twoshot or a ring")
        if op in LOC_OPS and algo == "nccl":
            raise ValueError(f"nccl has no maxloc or minloc: op={op} needs twoshot, a ring or ring-nccl")
        if op in ("min", "max") and algo in ("nccl", "ring-nccl") and dtype in UNSIGNED_TYPES:
            raise ValueError(f"{algo} compares {dtype} as a signed torch type: op={op} is refused")
        self.op = op
        self._op_kw = {} if op == "sum" else {"op": op}   # sum calls stay exactly as they were
        super().__init__(comm, device, native(), algo, ctas, _shared, VIRTUAL_ALGOS)
        self.dtype, self.chunk_elems = dtype, chunk_elems
        self.esz = self.C.elem_size(dtype)
        n = element_count(self.esz, self.world, log2_elems, n_elems)
        self.n, self.nbytes = n, n * self.esz
        self.right, self.left = (self.rank + 1) % self.world, (self.rank - 1) % self.world
        if slots not in (0, 2):
            raise ValueError("slots must be 0 (world-1 slots) or 2")
        self.slots_policy = slots if algo == "ring" else 0
        self.pull = bool(pull) and algo == "ring"
        self.n_chunks, pad_words, slot_bytes = _layout(algo, self.C, n, self.esz, self.world, chunk_elems,
                                                       self.slots_policy)
        self.ring_epoch = 0
        self.step_epoch = 0
        self.launches = 0
        self.va = self.vb = self.vc = self.slots = None
        self._symm = None
        if _shared is not None:         # virtual ranks of one process (VirtualAllreduce): buffers made by the group
            self.pads, self.va, self.vb, self.vc, self.slots = (_shared.get(k) for k in ("pads", "va", "vb", "vc",
                                                                                          "slots"))
        elif algo == "nvls":
            self.pads = SignalPads(comm, device, extra_words=pad_words, timeout_s=timeout_s)
            try:
                self._init_nvls()
            except Exception:
                self.pads.close()   # collectively allocated just above: do not leak it on the failure path
                raise
        else:
            self.pads = SignalPads(comm, device, extra_words=pad_words, timeout_s=timeout_s)
            self.va = SymmetricBuffer(comm, self.nbytes, device)
            self.vc = SymmetricBuffer(comm, self.nbytes, device)
            if algo in ("ring", "ring-rsag"):
                self.slots = SymmetricBuffer(comm, slot_bytes, device, zero=False)
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

    def _ptrs(self):
        if self.algo == "nvls":
            return self._va_ptr, self._vc_ptr
        return self.va.local_ptr, self.vc.local_ptr

    def initialize(self) -> None:
        va, vc = self._ptrs()
        vb = self.vb.local_ptr if self.vb is not None else 0
        if self.dtype in PAIR_TYPES:
            x, i = loc_input(self.op, self.rank, self.world)
            for p in (va, vb):
                if p:
                    self.C.init_pair(p, self.n, x, i, self.dtype, self._stream())
            self.C.init_pair(vc, self.n, *loc_vc_init(self.op), self.dtype, self._stream())
            return
        x = op_input(self.op, self.rank, self.world)
        # VC: 0 for the sum, which accumulates into it; the other ops must overwrite it whatever it holds
        self.C.init3(va, vb, vc, self.n, x, x, vc_init(self.op, self.world), self.dtype, self._stream())

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
                             self.slots.ptrs[self.left] if self.pull else 0, **self._op_kw)
            self.ring_epoch += P
            self.launches += 1
        elif self.algo == "ring-rsag":
            C.ring_rsag(va=va, vc=vc, slots_local=self.slots.local_ptr, slots_right=self.slots.ptrs[self.right],
                        vc_right=self.vc.ptrs[self.right], arrived_local=pads.chunk_word(me),
                        arrived_right=pads.chunk_word(self.right), rank=me, world=P, n=self.n,
                        chunk_elems=self.chunk_elems, epoch_base=self.ring_epoch, timeout_ns=pads.timeout_ns,
                        status=pads.status_ptr, dtype=self.dtype, ctas=self.ctas, device=self.device, stream=st,
                        phases="allreduce", **self._op_kw)
            self.ring_epoch += C.rsag_epoch_advance(C.RSAG_ALLREDUCE, P)
            self.launches += 1
        elif self.algo == "twoshot":
            pads.barrier_epoch += 1
            ctas = C.allreduce_two_shot(self.va.ptrs, self.vc.ptrs, pads.buf.ptrs, pads.ticket_ptr,
                                        pads.ticket_issued & 0xFFFFFFFF, me, self.n, pads.barrier_epoch,
                                        pads.timeout_ns, pads.status_ptr, self.dtype, self.ctas,
                                        self.device, st, **self._op_kw)
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
                dist.all_reduce(dst, **({"op": _nccl_op(self.op)} if self.op != "sum" else {}))
        elif self.algo == "ring-unfused":
            cur, other = va, self.vb.local_ptr
            r_other = self.vb.ptrs[self.right]
            r_cur = self.va.ptrs[self.right]
            if self.op == "sum":
                C.accumulate(cur, vc, self.n, self.dtype, st)
            else:                                       # the other ops overwrite VC: step 0 is VC = VA
                C.memcpy_async(vc, cur, self.nbytes, st)
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
                C.accumulate(cur, vc, self.n, self.dtype, st, **self._op_kw)
                self.launches += 4
            self.launches += 1
        elif self.algo == "ring-nccl":
            import torch.distributed as dist
            from ..parallel.symmetric import tensor_from_ptr
            td = _TORCH_DTYPE.get(self.dtype, torch.uint8)    # pair types: their bytes
            cur = tensor_from_ptr(va, self.nbytes, self.device, td)
            other = self.vb.tensor(td)
            acc = tensor_from_ptr(vc, self.nbytes, self.device, td)
            combine = {"sum": lambda: acc.add_(cur), "prod": lambda: torch.mul(acc, cur, out=acc),
                       "min": lambda: torch.minimum(acc, cur, out=acc),
                       "max": lambda: torch.maximum(acc, cur, out=acc),
                       "band": lambda: torch.bitwise_and(acc, cur, out=acc),
                       "bor": lambda: torch.bitwise_or(acc, cur, out=acc),
                       "bxor": lambda: torch.bitwise_xor(acc, cur, out=acc),
                       "land": lambda: acc.copy_(torch.logical_and(acc, cur).to(td)),
                       "lor": lambda: acc.copy_(torch.logical_or(acc, cur).to(td)),
                       "lxor": lambda: acc.copy_(torch.logical_xor(acc, cur).to(td)),
                       "maxloc": lambda: acc.copy_(loc_combine(acc, cur, self.dtype, "maxloc")),
                       "minloc": lambda: acc.copy_(loc_combine(acc, cur, self.dtype, "minloc"))}
            if self.op == "sum":
                acc.add_(cur)
            else:
                acc.copy_(cur)
            torch.cuda.synchronize(self.device)        # the reference's .wait()
            for _ in range(1, P):
                ops = [dist.P2POp(dist.isend, cur, self.right), dist.P2POp(dist.irecv, other, self.left)]
                for w in dist.batch_isend_irecv(ops):
                    w.wait()
                torch.cuda.synchronize(self.device)    # blocking MPI_Send/Recv semantics
                cur, other = other, cur
                combine[self.op]()
                torch.cuda.synchronize(self.device)

    def mismatches(self) -> int:
        _, vc = self._ptrs()
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        if self.dtype in PAIR_TYPES:
            self.C.count_pair_mismatch(vc, self.n, *loc_expected(self.op, self.world), self.dtype, count.data_ptr(),
                                       self._stream())
        else:
            self.C.count_mismatch(vc, self.n, expected_value(self.world, self.op), self.dtype, count.data_ptr(),
                                  self._stream())
        torch.cuda.synchronize(self.device)
        return int(count.item())

    def result(self, ms: float, mismatches: int) -> AllreduceResult:
        return AllreduceResult(self.algo, self.dtype, self.world, self.n, ms, mismatches, self.esz, self.op)


class VirtualAllreduce(VirtualRanks):
    """``world`` AllreduceMiniapp ranks on one GPU (``VirtualRanks``): the ring's arrival and ack words, the two-shot
    barrier and the unfused ring's rendezvous run on a 1-GPU box with the same ``run_once`` plumbing as one process per
    GPU.  The unfused ring launches a kernel for the first time next to spinning ones, which needs the eager module
    loading this package asks for when it is imported before CUDA starts."""

    def __init__(self, world: int, n: int, dtype: str = "float", algo: str = "ring", slots: int = 0,
                 pull: bool = False, ctas: int = 0, chunk_elems: int = 0, device: int = 0, timeout_s: float = 10.0,
                 op: str = "sum"):
        self.refuse(world, algo, VIRTUAL_ALGOS)
        op = reduce_op(op)
        check_op_type(op, dtype)
        C = native()
        esz = C.elem_size(dtype)
        n = element_count(esz, world, n_elems=n)
        super().__init__(world, device, ctas)
        self.dtype, self.n = dtype, n
        policy = slots if algo == "ring" else 0
        _, pad_words, slot_bytes = _layout(algo, C, n, esz, world, chunk_elems, policy)
        none = [None] * world
        pads = self.group.pads(extra_words=pad_words, timeout_s=timeout_s)
        va = self.group.symmetric(n * esz)
        vc = self.group.symmetric(n * esz)
        vb = self.group.symmetric(n * esz) if algo == "ring-unfused" else none
        sl = self.group.symmetric(slot_bytes, zero=False) if algo in ("ring", "ring-rsag") else none
        self.ranks: List[AllreduceMiniapp] = [
            AllreduceMiniapp(self.group.comms[r], device, dtype=dtype, algo=algo, chunk_elems=chunk_elems,
                             ctas=self.ctas, timeout_s=timeout_s, slots=slots, pull=pull, n_elems=n, op=op,
                             _shared={"pads": pads[r], "va": va[r], "vb": vb[r], "vc": vc[r], "slots": sl[r]})
            for r in range(world)]

    def load(self, vas: List[torch.Tensor]) -> None:
        """VA of rank r <- ``vas[r]`` (n elements of the dtype's torch type; for a pair type a (values, indices) tuple,
        packed by ``pack_loc``), VC <- 0 (the sum rings accumulate into it; ring-rsag and every op other than the sum
        overwrite it)."""
        torch.cuda.synchronize(self.device)
        for app, v in zip(self.ranks, vas):
            if self.dtype in PAIR_TYPES:
                app.va.tensor(torch.uint8).copy_(pack_loc(*v, dtype=self.dtype))
                app.vc.tensor(torch.uint8).zero_()
            else:
                app.va.tensor(_TORCH_DTYPE[self.dtype]).copy_(v)
                app.vc.tensor(_TORCH_DTYPE[self.dtype]).zero_()
        torch.cuda.synchronize(self.device)

    def results(self) -> List[torch.Tensor]:
        """VC of every rank, on the host; for a pair type a (values, int32 indices) tuple per rank (``unpack_loc``)."""
        self.synchronize()
        if self.dtype in PAIR_TYPES:
            return [unpack_loc(app.vc.tensor(torch.uint8).cpu(), self.dtype) for app in self.ranks]
        return [app.vc.tensor(_TORCH_DTYPE[self.dtype]).cpu() for app in self.ranks]


# -------------------------------------------------------------------------------------------------- reduce-scatter ----
# ``ReduceScatterMiniapp`` is the Python twin of ``bin/reduce_scatter`` (↔ MPI_Reduce_scatter_block, ncclReduceScatter):
# rank p's send buffer holds P segments of n elements, and afterwards rank r's receive buffer holds op over p of
# segment r of rank p's, owner first (``ops.allreduce.reduce_scatter``).  Algorithms: ``direct`` (one launch per rank,
# peer loads, default) and ``nccl`` (torch.distributed.reduce_scatter_tensor, sum / prod / min / max, the baseline).
RS_ALGOS = ("direct", "nccl")
RS_SUM_POISON = 251.0       # above every rank's constant-data sum up to 16 ranks (at most 232) and exact in every type


def rs_input(op: str, rank: int, segment: int, world: int) -> float:
    """What segment ``segment`` of ``rank``'s send buffer holds in the constant-data run: for the sum rank + (segment
    mod 8), so a rank that reduced another's segment gets another value; for the other ops the allreduce's
    ``op_input``."""
    return float(rank + segment % 8) if op == "sum" else op_input(op, rank, world)


def rs_expected(op: str, rank: int, world: int) -> float:
    """Every element of ``rank``'s receive buffer after the constant-data run."""
    return world * (world - 1) / 2.0 + world * (rank % 8) if op == "sum" else expected_value(world, op)


def rs_poison(op: str, world: int) -> float:
    """The receive buffer before the run: a value no rank expects (vc_init's 0 is rank 0's sum at one rank)."""
    return RS_SUM_POISON if op == "sum" else vc_init(op, world)


@dataclass
class ReduceScatterResult:
    algo: str
    dtype: str
    world: int
    elements: int        # per segment
    ms: float
    mismatches: int
    elem_bytes: int = 4
    op: str = "sum"

    def row(self) -> dict:
        """One JSON row; GB/s counts the (P-1) segments that leave every rank's send buffer for their owners."""
        sent = float(self.world - 1) * self.elements * self.elem_bytes
        return {"pattern": "reduce_scatter", "algo": self.algo, "type": self.dtype, "op": self.op,
                "ranks": self.world, "elements": self.elements, "ms": self.ms,
                "GBps_sent_per_rank": gbps(sent, self.ms), "mismatches": self.mismatches}


class ReduceScatterMiniapp(CollectiveMiniapp):
    PATTERN, UNIT = "reduce_scatter", "elements"

    def __init__(self, comm: Comm, device: int, log2_elems: int = 25, dtype: str = "float", op: str = "sum",
                 algo: str = "direct", ctas: int = 0, timeout_s: float = 30.0, n_elems: int = 0,
                 _shared: Optional[dict] = None):
        """The send buffer holds 2^log2_elems elements padded to P whole 16-byte segments (``n_elems``: exactly that
        many per rank).  ``_shared``: buffers made by an in-process group (``VirtualReduceScatter``): ``pads``,
        ``send``, ``recv``.  Every refusal is raised before anything is allocated."""
        if algo not in RS_ALGOS:
            raise ValueError(f"algo must be one of {RS_ALGOS}")
        if dtype not in DTYPES:
            raise ValueError(f"dtype must be one of {sorted(DTYPES)}")
        op = reduce_op(op)
        check_op_type(op, dtype)
        if algo == "nccl" and (op not in ("sum", "prod", "min", "max") or dtype in PAIR_TYPES):
            raise ValueError(f"nccl reduce-scatters sum, prod, min and max only: op={op} needs direct")
        if algo == "nccl" and op in ("min", "max") and dtype in UNSIGNED_TYPES:
            raise ValueError(f"nccl compares {dtype} as a signed torch type: op={op} is refused")
        super().__init__(comm, device, native(), algo, ctas, _shared, ("direct",))
        self.esz = self.C.elem_size(dtype)
        total = element_count(self.esz, self.world, log2_elems, n_elems)
        check_reduce_scatter_args(self.world, total // self.world, dtype)
        self.dtype, self.op = dtype, op
        self.n = total // self.world                 # elements per segment
        self.seg_bytes = self.n * self.esz
        if _shared is not None:
            self.pads, self.send, self.recv = _shared["pads"], _shared["send"], _shared["recv"]
        else:
            self.pads = SignalPads(comm, device, timeout_s=timeout_s)
            self.send = SymmetricBuffer(comm, self.world * self.seg_bytes, device, zero=False)
            self.recv = SymmetricBuffer(comm, self.seg_bytes, device, zero=False)   # only the local mapping is used

    def _tensor(self, buf: torch.Tensor) -> torch.Tensor:
        return buf if self.dtype in PAIR_TYPES else buf.view(_TORCH_DTYPE[self.dtype])

    def initialize(self) -> None:
        """The constant-data run's send segments and the poisoned receive buffer."""
        st, base = self._stream(), self.send.local_ptr
        for q in range(self.world):
            at = base + q * self.seg_bytes
            if self.dtype in PAIR_TYPES:
                self.C.init_pair(at, self.n, *loc_input(self.op, self.rank, self.world), self.dtype, st)
            else:
                x = rs_input(self.op, self.rank, q, self.world)
                self.C.init3(at, 0, 0, self.n, x, 0.0, 0.0, self.dtype, st)
        if self.dtype in PAIR_TYPES:
            self.C.init_pair(self.recv.local_ptr, self.n, *loc_vc_init(self.op), self.dtype, st)
        else:
            self.C.init3(self.recv.local_ptr, 0, 0, self.n, rs_poison(self.op, self.world), 0.0, 0.0, self.dtype, st)

    def run_once(self) -> None:
        """Enqueue one reduce-scatter on the current stream.  Precondition: every rank's send buffer is final and no
        rank still reads its receive buffer (``run()`` puts ``pads.device_barrier`` before it)."""
        pads, st = self.pads, self._stream()
        if self.algo == "nccl":
            import torch.distributed as dist
            src, dst = self._tensor(self.send.tensor()), self._tensor(self.recv.tensor())
            if self.world > 1:
                dist.reduce_scatter_tensor(dst, src, op=_nccl_op(self.op))
            else:
                dst.copy_(src)
            return
        pads.barrier_epoch += 1
        self.launch_ctas = reduce_scatter(self.send.ptrs, self.recv.local_ptr, pads.buf.ptrs, pads.ticket_ptr,
                                          pads.ticket_issued, self.rank, self.n, pads.barrier_epoch, pads.timeout_ns,
                                          pads.status_ptr, self.dtype, self.ctas, self.device, st, self.op)
        pads.advance_tickets(self.launch_ctas)

    def reduce_scatter(self, x: torch.Tensor) -> torch.Tensor:
        """Reduce-scatter the tensor ``x`` (P*n elements of the dtype, or its packed pairs): copy it into the symmetric
        send buffer, the device barrier and the launch, all enqueued on the current stream; returns this rank's n
        elements as a view of the receive buffer, which the next call overwrites.  Never synchronises the host."""
        xb = x.contiguous().view(torch.uint8).reshape(-1)
        if xb.numel() != self.world * self.seg_bytes:
            raise ValueError(f"reduce-scatter: x must hold {self.world} x {self.n} {self.dtype} elements")
        self.send.tensor().copy_(xb)
        if self.algo != "nccl":
            self.pads.device_barrier(self._stream())
        self.run_once()
        return self._tensor(self.recv.tensor())

    def mismatches(self) -> int:
        """Wrong elements of the receive buffer after the constant-data run, plus those of the send buffer (which must
        be unchanged)."""
        count = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.device))
        st, c = self._stream(), count.data_ptr()
        for q in range(self.world):
            at = self.send.local_ptr + q * self.seg_bytes
            if self.dtype in PAIR_TYPES:
                self.C.count_pair_mismatch(at, self.n, *loc_input(self.op, self.rank, self.world), self.dtype, c, st)
            else:
                self.C.count_mismatch(at, self.n, rs_input(self.op, self.rank, q, self.world), self.dtype, c, st)
        if self.dtype in PAIR_TYPES:
            self.C.count_pair_mismatch(self.recv.local_ptr, self.n, *loc_expected(self.op, self.world), self.dtype,
                                       c, st)
        else:
            self.C.count_mismatch(self.recv.local_ptr, self.n, rs_expected(self.op, self.rank, self.world),
                                  self.dtype, c, st)
        torch.cuda.synchronize(self.device)
        return int(count.item())

    def result(self, ms: float, mismatches: int) -> ReduceScatterResult:
        return ReduceScatterResult(self.algo, self.dtype, self.world, self.n, ms, mismatches, self.esz, self.op)


class VirtualReduceScatter(VirtualRanks):
    """``world`` ReduceScatterMiniapp ranks on one GPU (``VirtualRanks``).  ``n`` is the segment, in elements."""

    def __init__(self, world: int, n: int, dtype: str = "float", op: str = "sum", ctas: int = 0, device: int = 0,
                 timeout_s: float = 10.0):
        self.refuse(world)
        if dtype not in DTYPES:
            raise ValueError(f"dtype must be one of {sorted(DTYPES)}")
        op = reduce_op(op)
        check_op_type(op, dtype)
        check_reduce_scatter_args(world, n, dtype)
        C = native()
        super().__init__(world, device, ctas)
        self.n, self.dtype, self.op = int(n), dtype, op
        pads = self.group.pads(timeout_s=timeout_s)
        send = self.group.symmetric(world * self.n * C.elem_size(dtype), zero=False)
        recv = self.group.symmetric(self.n * C.elem_size(dtype), zero=False)
        self.ranks: List[ReduceScatterMiniapp] = [
            ReduceScatterMiniapp(self.group.comms[r], device, dtype=dtype, op=op, ctas=self.ctas, timeout_s=timeout_s,
                                 n_elems=world * self.n, _shared={"pads": pads[r], "send": send[r], "recv": recv[r]})
            for r in range(world)]

    def load(self, sends: List[torch.Tensor]) -> None:
        """Send buffer of rank r <- ``sends[r]``: P*n elements of the dtype's torch type, or any tensor of as many
        bytes (a pair type's packed bytes)."""
        if len(sends) != self.world:
            raise ValueError(f"one send tensor per rank ({self.world})")
        torch.cuda.synchronize(self.device)
        for app, s in zip(self.ranks, sends):
            b = s.contiguous().view(torch.uint8).reshape(-1)
            if b.numel() != self.world * app.seg_bytes:
                raise ValueError(f"a send tensor must hold {self.world} x {self.n} {self.dtype} elements")
            app.send.tensor().copy_(b)
        torch.cuda.synchronize(self.device)

    def results(self) -> List[torch.Tensor]:
        """The receive buffer of every rank on the host (n elements; a pair type's packed bytes)."""
        self.synchronize()
        return [app._tensor(app.recv.tensor()).cpu() for app in self.ranks]


def main_reduce_scatter(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200 reduce_scatter [-p K] [--type T] [--op OP]
    [--algo direct|nccl]``"""
    import argparse

    ap = argparse.ArgumentParser(prog="reduce_scatter", add_help=True)
    ap.add_argument("-p", "--log2-elems", type=int, default=25, help="2^K elements of send buffer per rank")
    ap.add_argument("--type", default="float", choices=DTYPES)
    ap.add_argument("--op", default="sum")
    ap.add_argument("--algo", default="direct", choices=RS_ALGOS)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ctas", type=int, default=0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args(argv)
    check_op_type(reduce_op(args.op), args.type)
    comm = Comm()
    app = ReduceScatterMiniapp(comm, comm.device, args.log2_elems, args.type, args.op, args.algo, ctas=args.ctas)
    res = app.run(args.iters, args.warmup)
    return report(comm, app, res, args, f"reduce_scatter {args.algo} {args.type} {app.op} P={comm.world} n={app.n}")


def choose_collective(comm: Comm, device: int, dtype: str, log2_elems: int, op: str = "sum"):
    """Which one-launch collective the ``-a`` path (↔ MPI_Allreduce, allreduce-mpi-sycl.cpp:61-67) uses.

    Decided BEFORE anything is allocated and agreed across ranks (min over ranks of the local probe), so ranks can
    neither diverge on the algorithm nor leak a half-built instance:
      * int:   two-shot — ``multimem.ld_reduce`` has no vector form for .s32 (one 4-byte request per thread), peer loads are 128-bit for every type;
      * bfloat16 / half: two-shot — its fp32 accumulation rounds once, where the rings round P-1 times (the NVLS
        kernel reduces fp32 and 32-bit integers only);
      * float: NVLS (in-switch reduction) when every rank reports multicast support, else two-shot;
      * any op but the sum: two-shot (the NVLS kernel reduces sums only)."""
    C = native()
    if reduce_op(op) != "sum":
        return "twoshot", f"op={reduce_op(op)}: NVLS reduces sums only"
    if dtype in FLOAT16_TYPES:
        return "twoshot", "16-bit floats: two-shot sums in fp32 and rounds once"
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
    ap.add_argument("--type", default="float", choices=sorted(DTYPES))
    ap.add_argument("--algo", default="ring", choices=ALGOS)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None)
    ap.add_argument("--slots", type=int, default=0, choices=(0, 2),
                    help="fused ring: 2 = two receive slots + per-chunk acks (VA/VB double buffer); "
                         "default world-1 slots")
    ap.add_argument("--pull", action="store_true",
                    help="fused ring, receiver-driven: blocks are loaded from the left neighbour (peer loads)")
    ap.add_argument("--op", default=None, choices=OPS + tuple(_OP_ALIASES),
                    help="reduction (default sum, maxloc on a pair type; nvls is sum-only, -a uses two-shot for the "
                         "others; band bor bxor land lor lxor take integer types only, maxloc minloc pair types only)")
    args = ap.parse_args(argv)
    op = reduce_op(args.op if args.op is not None else "maxloc" if args.type in PAIR_TYPES else "sum")
    check_op_type(op, args.type)
    comm = Comm()
    device = comm.device   # chosen before the process group was bound to it (Comm.pick_device)
    algo = args.algo
    app = None
    if args.a:
        algo, why = choose_collective(comm, device, args.type, args.p, op)
        if comm.rank == 0:
            print(f"# -a: {algo} ({why})", flush=True)
    app = AllreduceMiniapp(comm, device, args.p, args.type, algo, slots=args.slots, pull=args.pull, op=op)
    res = app.run(args.iters, args.warmup)
    return report(comm, app, res, args,
                  f"{algo} {args.type} P={comm.world} N={res.elements}{'' if op == 'sum' else ' op=' + op}")


if __name__ == "__main__":
    raise SystemExit(main())
