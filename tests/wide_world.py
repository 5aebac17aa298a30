"""Collectives at 9 to 16 ranks on ONE GPU: the ranks' launches run one after another on a single stream.

The two-shot allreduce, the reduce-scatter, the all-to-all, the all-gather and the all-to-all-v each end with one
cross-rank wait, the node barrier of ``grid_then_node_barrier`` (csrc/kernels/ring_allreduce.cuh): lane t < P of the
last CTA stores the epoch into word ``rank`` of rank t's barrier section and waits for word t of its own.  Before that
wait a grid reads only inputs no rank writes during the launch (VA, the send buffers, the counts) and writes disjoint
outputs.  So the P launches can run serially, with no co-residency and no extra hardware queue, as long as each rank's
barrier finds its peers' words already reached:

* ``SerialRanks.arm(e)`` writes e + 2^30 into words [0, P) of every rank's barrier section before the launches of
  epoch e.  ``epoch_reached`` compares (int32)(seen - want) >= 0, so these count as reached, and no kernel ever waits;
* every kernel overwrites the words it owns with exactly e, so ``check_arrivals(e)`` finds each rank's arrival: word t
  of every pad must hold e (a rank that never arrives, or arrives in another rank's word, leaves e + 2^30 behind),
  words P..15 stay untouched, every status word reads OK and every ticket word equals what the host issued.

A TIMEOUT status is therefore a finding to explain, never something to retry.  What this does not exercise is 9 or
more grids spinning on each other at once: that code (``threadIdx.x < world`` inside warp 0) is the one <= 8 ranks run.

The drivers below run three launches of one collective with fresh data and an advancing epoch, every output poisoned
first, and check every rank bit for bit against the suite's oracles, its guards, its unchanged inputs and the arrival
words.  A launch's problems are raised together as one ``WideWorldError`` that names the launch, the rank and the first
wrong element; ``.ranks`` holds the ranks it names.  Nothing here needs a GPU: tests/test_wide_worlds_emulated.py runs
the same drivers on the emulated device (tests/wide_world_emu.py), tests/test_gpu_wide_worlds.py on an H100.
"""
from __future__ import annotations

from typing import Callable, List, Tuple

import torch

import tests.allreduce_oracle as aro
import tests.alltoallv_oracle as a2av
import tests.bitop_oracle as bit
import tests.loc_oracle as loc
import tests.lowp_allreduce_oracle as lowp
import tests.reduce_op_oracle as rop
import tests.reduce_scatter_oracle as rso
from hpc_patterns_b200.ops.alltoall import all_to_all_reference, all_to_all_v_reference
from hpc_patterns_b200.parallel.local import LocalGroup

ARM = 1 << 30               # added to the epoch in the pre-armed barrier words
MAX_RANKS = 16              # words per barrier section (kMaxRanks, csrc/common/signal_layout.h)
TIMEOUT_S = 5.0             # no kernel waits: a deadline of a few seconds only bounds a broken arming
LAUNCHES = 3
GUARD = 64                  # elements (or bytes, for the byte-moving collectives) after every output, never written
MASK = 0xFFFFFFFF

Problems = List[Tuple[int, str]]


class WideWorldError(AssertionError):
    """Everything wrong with one launch; ``ranks`` are the ranks the problems name."""

    def __init__(self, launch: int, problems: Problems):
        self.launch = launch
        self.ranks = sorted({r for r, _ in problems})
        super().__init__(f"launch {launch}: " + "; ".join(f"rank {r}: {what}" for r, what in problems))


class SerialRanks:
    """``world`` virtual ranks on one device whose launches run in rank order on ONE stream, with pre-armed barriers
    (module docstring).  Buffers and pads come from ``LocalGroup(world, [device] * world)``."""

    def __init__(self, world: int, device: int = 0, timeout_s: float = TIMEOUT_S):
        if not 1 <= world <= MAX_RANKS:
            raise ValueError(f"serial ranks: 1 <= world <= {MAX_RANKS}")
        self.world, self.device = world, device
        self.group = LocalGroup(world, [device] * world)
        self.pads = self.group.pads(timeout_s=timeout_s)
        self.C = self.pads[0].C
        self.stream = torch.cuda.Stream(device)
        self.epoch = 0
        self._buffers = []

    @property
    def pad_ptrs(self) -> List[int]:
        return self.pads[0].buf.ptrs

    def symmetric(self, nbytes: int):
        """One buffer of ``nbytes`` per rank (zeroed), freed by ``close``."""
        b = self.group.symmetric(nbytes, zero=True)
        self._buffers.append(b)
        return b

    def _pad(self, rank: int) -> torch.Tensor:
        return self.pads[rank].buf.tensor(torch.int32)

    def arm(self, epoch: int) -> None:
        """Words [0, P) of every barrier section hold epoch + 2^30: reached for every wait of this epoch."""
        b = self.C.PAD_BARRIER
        for r in range(self.world):
            self._pad(r)[b:b + self.world].fill_(epoch + ARM)

    def launch(self, enqueue: Callable[[int, int], int]) -> Problems:
        """One collective of the next epoch e: ``arm(e)``, then ``enqueue(rank, e)`` for rank 0, 1, ... on the one
        stream (it returns the CTAs launched; the rank's tickets advance by them), one synchronise, and the problems
        ``check_arrivals(e)`` finds."""
        e = self.epoch + 1
        torch.cuda.synchronize(self.device)             # the data loads of the default stream
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            self.arm(e)
            for r, p in enumerate(self.pads):
                p.barrier_epoch = e
                p.advance_tickets(enqueue(r, e))
        self.stream.synchronize()
        self.epoch = e
        return self.check_arrivals(e)

    def check_arrivals(self, epoch: int) -> Problems:
        """Every rank arrived in its own word of every pad, nothing else in the barrier sections changed, every status
        word is OK and every ticket word counts exactly the CTAs issued."""
        C, P, b = self.C, self.world, self.C.PAD_BARRIER
        words = [[w & MASK for w in self._pad(r).cpu().tolist()] for r in range(P)]
        problems = []
        for t in range(P):
            missing = [r for r in range(P) if words[r][b + t] != epoch]
            if missing:
                problems.append((t, f"no arrival of epoch {epoch} in barrier word {t} of the pads of ranks {missing} "
                                    f"(rank {missing[0]}'s holds {words[missing[0]][b + t]:#x})"))
        for r, w in enumerate(words):
            stray = [t for t in range(P, MAX_RANKS) if w[b + t] != 0]
            if stray:
                problems.append((r, f"barrier words {stray} of its pad were written (no rank >= {P} exists)"))
            status = w[C.PAD_WORDS + self.pads[r].extra_words]
            if status != C.STATUS_OK:
                kind = "TIMEOUT" if status == C.STATUS_TIMEOUT else f"{status:#010x}"
                problems.append((r, f"status word {kind} (no kernel should ever wait here)"))
            ticket = w[C.PAD_LOCAL]
            if ticket != self.pads[r].ticket_issued & MASK:
                problems.append((r, f"ticket word {ticket}, the host issued {self.pads[r].ticket_issued & MASK}"))
        return problems

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        for b in self._buffers:
            for x in b:
                x.close()
        self._buffers = []
        for p in self.pads:
            p.close()
        self.pads = []


# ------------------------------------------------------------------------------------------------------- helpers ----
def elem_bytes(dtype: str) -> int:
    return loc.pair_bytes(dtype) if dtype in loc.PAIR_TYPES else rop.elem_bytes(dtype)


def as_bytes(x) -> torch.Tensor:
    """A CPU uint8 tensor of the bytes of ``x`` (a tensor of any dtype, or bytes)."""
    if isinstance(x, (bytes, bytearray)):
        return torch.frombuffer(bytearray(x), dtype=torch.uint8)
    return x.detach().contiguous().view(torch.uint8).reshape(-1).cpu()


def first_wrong(got: torch.Tensor, want: torch.Tensor, esz: int, base: int = 0) -> str:
    """'' if the bytes are equal, else how many ``esz``-byte elements differ and the first one (index + ``base``)."""
    differ = (got != want).reshape(-1, esz).any(1)
    if not bool(differ.any()):
        return ""
    i = int(differ.nonzero()[0])
    g, w = (bytes(t[i * esz:(i + 1) * esz].tolist()).hex() for t in (got, want))
    return f"{int(differ.sum())} wrong elements, first [{base + i}]: bytes {g}, want {w}"


def _raise(launch: int, problems: Problems) -> None:
    if problems:
        raise WideWorldError(launch, problems)


def two_shot_expected(vas, op: str, dtype: str):
    """VC of every rank after a two-shot allreduce of ``vas`` (bytes for a pair type): the pinned order for the float
    and double sum, else the fold of the oracle that owns (op, dtype)."""
    if op == "sum":
        if dtype in aro.FLOATING:
            return aro.two_shot_sum_pinned(vas)
        if dtype in lowp.LOWP:
            return lowp.two_shot_expected(vas)
        return aro.ring_expected(vas, 0)                 # integers: the wrapping sum, in any order
    if dtype in loc.PAIR_TYPES:
        return loc.allreduce_expected(op, vas, dtype)
    if op in bit.BIT_OPS:
        return bit.allreduce_expected(vas, op, dtype)
    return rop.two_shot_expected(vas, op, dtype)


def _seed(*xs) -> int:
    return sum(x * 1009 ** k for k, x in enumerate(xs)) % (1 << 31)


# ------------------------------------------------------------------------------------------------------ two-shot ----
def two_shot(sr: SerialRanks, dtype: str, op: str, slice_vec: int, ctas: int = 0, launches: int = LAUNCHES,
             seed: int = 0) -> None:
    """``allreduce_two_shot`` with slices of ``slice_vec`` 16-byte vectors: every rank's VC bit-equal to
    ``two_shot_expected``, VC poisoned with 0xFF before and followed by GUARD untouched elements, VA unchanged."""
    C, P = sr.C, sr.world
    esz = elem_bytes(dtype)
    per = slice_vec * 16 // esz
    n, nb = per * P, per * P * esz
    va, vc = sr.symmetric(nb), sr.symmetric(nb + GUARD * esz)
    guard = torch.randint(0, 256, (GUARD * esz,), dtype=torch.uint8,
                          generator=torch.Generator().manual_seed(_seed(P, slice_vec, seed)))
    for launch in range(launches):
        vas = rso.make_inputs(P, per, dtype, op, seed=_seed(P, slice_vec, seed), launch=launch)
        raw = [as_bytes(v) for v in vas]
        for r in range(P):
            va[r].tensor().copy_(raw[r])
            vc[r].tensor()[:nb].fill_(0xFF)
            vc[r].tensor()[nb:].copy_(guard)

        def enqueue(r, e):
            p = sr.pads[r]
            return C.allreduce_two_shot(va[r].ptrs, vc[r].ptrs, sr.pad_ptrs, p.ticket_ptr, p.ticket_issued & MASK, r,
                                        n, e, p.timeout_ns, p.status_ptr, dtype, ctas, sr.device,
                                        sr.stream.cuda_stream, op)

        problems = sr.launch(enqueue)
        want = as_bytes(two_shot_expected(vas, op, dtype))
        got = [vc[r].tensor().cpu() for r in range(P)]
        sb = per * esz
        for s in range(P):                  # slice s is rank s's reduction, stored into every rank's VC
            bad = [(r, first_wrong(got[r][s * sb:(s + 1) * sb], want[s * sb:(s + 1) * sb], esz, s * per))
                   for r in range(P)]
            bad = [(r, why) for r, why in bad if why]
            if bad:
                problems.append((s, f"its slice is wrong in the VC of ranks {[r for r, _ in bad]}; "
                                    f"rank {bad[0][0]}'s VC: {bad[0][1]}"))
        for r in range(P):
            if not torch.equal(got[r][nb:], guard):
                problems.append((r, "a guard element after its VC was written"))
            if not torch.equal(va[r].tensor().cpu(), raw[r]):
                problems.append((r, "its VA changed"))
        _raise(launch, problems)


# ------------------------------------------------------------------------------------------------ reduce-scatter ----
def reduce_scatter(sr: SerialRanks, dtype: str, op: str, seg_vec: int, ctas: int = 0, launches: int = LAUNCHES,
                   seed: int = 0) -> None:
    """``reduce_scatter`` with segments of ``seg_vec`` vectors: every receive buffer bit-equal to
    ``reduce_scatter_oracle.expected``, poisoned before and followed by GUARD untouched elements, sends unchanged."""
    C, P = sr.C, sr.world
    esz = elem_bytes(dtype)
    n = seg_vec * 16 // esz
    sb = n * esz
    send, recv = sr.symmetric(P * sb), sr.symmetric(sb + GUARD * esz)
    for launch in range(launches):
        sends = rso.make_inputs(P, n, dtype, op, seed=_seed(P, seg_vec, seed), launch=launch)
        raw = [as_bytes(s) for s in sends]
        for r in range(P):
            send[r].tensor().copy_(raw[r])
            recv[r].tensor().fill_(0xA5 ^ launch)

        def enqueue(r, e):
            p = sr.pads[r]
            return C.reduce_scatter(send[r].ptrs, recv[r].local_ptr, sr.pad_ptrs, p.ticket_ptr, p.ticket_issued & MASK,
                                    r, n, e, p.timeout_ns, p.status_ptr, dtype, ctas, sr.device, sr.stream.cuda_stream,
                                    op)

        problems = sr.launch(enqueue)
        for r in range(P):
            got = recv[r].tensor().cpu()
            why = first_wrong(got[:sb], as_bytes(rso.expected(sends, r, op, dtype)), esz)
            if why:
                problems.append((r, f"receive buffer: {why}"))
            if not bool((got[sb:] == (0xA5 ^ launch)).all()):
                problems.append((r, "a guard element after its receive buffer was written"))
            if not torch.equal(send[r].tensor().cpu(), raw[r]):
                problems.append((r, "its send buffer changed"))
        _raise(launch, problems)


# ----------------------------------------------------------------------------------------- all-to-all, all-gather ----
def _random_bytes(count: int, nbytes: int, seed: int) -> List[torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (nbytes,), dtype=torch.uint8, generator=g) for _ in range(count)]


def _moved(sr: SerialRanks, name: str, block_bytes: int, pull: bool, ctas: int, launches: int, seed: int) -> None:
    C, P, B = sr.C, sr.world, block_bytes
    gather = name == "all_gather"
    sb = B if gather else P * B
    send, recv = sr.symmetric(sb), sr.symmetric(P * B + GUARD)
    for launch in range(launches):
        sends = _random_bytes(P, sb, _seed(P, B, int(pull), seed, launch))
        for r in range(P):
            send[r].tensor().copy_(sends[r])
            recv[r].tensor().fill_(0x5A ^ launch)

        def enqueue(r, e):
            p = sr.pads[r]
            return getattr(C, name)(send[r].ptrs, recv[r].ptrs, sr.pad_ptrs, p.ticket_ptr, p.ticket_issued & MASK, r,
                                    B, e, p.timeout_ns, p.status_ptr, ctas, sr.device, sr.stream.cuda_stream, pull)

        problems = sr.launch(enqueue)
        want = [torch.stack(sends)] * P if gather else all_to_all_reference(sends)
        for r in range(P):
            got = recv[r].tensor().cpu()
            for p in range(P):
                why = first_wrong(got[p * B:(p + 1) * B], want[r][p], 1)
                if why:
                    problems.append((r, f"block {p} (from rank {p}): {why}"))
            if not bool((got[P * B:] == (0x5A ^ launch)).all()):
                problems.append((r, "a guard byte after its receive buffer was written"))
            if not torch.equal(send[r].tensor().cpu(), sends[r]):
                problems.append((r, "its send buffer changed"))
        _raise(launch, problems)


def all_to_all(sr: SerialRanks, block_bytes: int, pull: bool, ctas: int = 0, launches: int = LAUNCHES,
               seed: int = 0) -> None:
    """``all_to_all`` of random bytes: block p of rank r's receive buffer is block r of rank p's send buffer."""
    _moved(sr, "all_to_all", block_bytes, pull, ctas, launches, seed)


def all_gather(sr: SerialRanks, block_bytes: int, pull: bool, ctas: int = 0, launches: int = LAUNCHES,
               seed: int = 0) -> None:
    """``all_gather`` of random bytes: every receive buffer is the concatenation of the send blocks."""
    _moved(sr, "all_gather", block_bytes, pull, ctas, launches, seed)


# ---------------------------------------------------------------------------------------------------- all-to-all-v ----
MEAN = 24                   # mean rows per pair: capacities of 2 * P * MEAN rows


class AllToAllV:
    """``all_to_all_v`` on ``sr`` with rows of ``row_bytes``.  Declared send and receive capacities are ``cap`` rows;
    twice that is allocated, so a kernel that ignored a refusal would still write inside its buffers, onto poison."""

    def __init__(self, sr: SerialRanks, row_bytes: int, pull: bool, mean: int = MEAN):
        P = sr.world
        self.sr, self.R, self.pull = sr, row_bytes, pull
        self.cap = 2 * P * mean
        self.rows = 2 * self.cap
        self.send, self.recv = sr.symmetric(self.rows * row_bytes), sr.symmetric(self.rows * row_bytes)
        self.counts, self.recv_counts = sr.symmetric(8 * P), sr.symmetric(8 * P)
        self.verdict = sr.symmetric(16)

    def launch(self, m, launch: int, seed: int = 0) -> None:
        """One launch of the count matrix ``m`` (P lists of P ints) with fresh bytes: an accepted matrix must move
        exactly ``all_to_all_v_reference``'s rows, a refused one no byte; every rank reports the oracle's verdict and
        its exact column as recv_counts."""
        sr, C, P, R = self.sr, self.sr.C, self.sr.world, self.R
        sends = _random_bytes(P, self.rows * R, _seed(P, R, int(self.pull), seed, launch))
        for r in range(P):
            self.send[r].tensor().copy_(sends[r])
            self.counts[r].tensor(torch.int64).copy_(torch.tensor(m[r], dtype=torch.int64))
            self.recv[r].tensor().fill_(0x5A ^ launch)
            self.recv_counts[r].tensor(torch.int64).fill_(-7)
            self.verdict[r].tensor(torch.int32).fill_(-1)

        def enqueue(r, e):
            p = sr.pads[r]
            return C.all_to_all_v(self.send[r].ptrs, self.recv[r].ptrs, self.counts[r].ptrs,
                                  self.recv_counts[r].local_ptr, self.verdict[r].local_ptr, sr.pad_ptrs, p.ticket_ptr,
                                  p.ticket_issued & MASK, r, R, self.cap, self.cap, e, p.timeout_ns, p.status_ptr, 0,
                                  sr.device, sr.stream.cuda_stream, self.pull)

        problems = sr.launch(enqueue)
        rule = a2av.verdict(m, self.cap, self.cap)
        want = all_to_all_v_reference(sends, m, R) if rule == 0 else [torch.empty(0, R, dtype=torch.uint8)] * P
        for r in range(P):
            verdict = self.verdict[r].tensor(torch.int32)[0].item() & MASK
            if verdict != rule:
                problems.append((r, f"verdict {verdict}, the rules give {rule}"))
            rc = self.recv_counts[r].tensor(torch.int64).cpu().tolist()
            if rc != [m[p][r] for p in range(P)]:
                problems.append((r, f"recv_counts {rc}, want {[m[p][r] for p in range(P)]}"))
            got = self.recv[r].tensor().cpu()
            total = want[r].numel()
            why = first_wrong(got[:total], want[r].reshape(-1), R)
            if why:
                problems.append((r, f"received rows: {why}"))
            if not bool((got[total:] == (0x5A ^ launch)).all()):
                k = int((got[total:] != (0x5A ^ launch)).nonzero()[0]) // R + total // R
                problems.append((r, f"row {k}, past the {total // R} rows it receives, was written"
                                    + (" (a refused launch)" if rule else "")))
            if not torch.equal(self.send[r].tensor().cpu(), sends[r]):
                problems.append((r, "its send buffer changed"))
            if self.counts[r].tensor(torch.int64).cpu().tolist() != list(m[r]):
                problems.append((r, "its counts changed"))
        _raise(launch, problems)

    def refused(self, rule: int):
        """A matrix that breaks ``rule`` (1 negative count, 2 send capacity, 3 receive capacity) only in the last row
        (rules 1, 2) or the last column (rule 3): at 9 or more ranks, an entry no <= 8-rank judge thread reads."""
        P, cap, last = self.sr.world, self.cap, self.sr.world - 1
        m = [[MEAN // 2] * P for _ in range(P)]
        if rule == a2av.NEGATIVE:
            m[last][3] = -1
        elif rule == a2av.SEND_CAPACITY:
            m[last] = [cap // P + 3] * P
        elif rule == a2av.RECV_CAPACITY:
            for p in range(P):
                m[p][last] = cap // P + 2
        assert a2av.verdict(m, cap, cap) == rule
        return m
