"""Virtual ranks inside one process: several "ranks" on one GPU, or one process driving several GPUs.

The reference fakes a larger machine only by oversubscription — more MPI ranks than devices, dealt
round-robin (aurora.mpich.miniapps/src/include/devices.hpp:46-47).  The native CLIs here do the same
with their thread-per-rank runtime.  ``LocalGroup`` is the Python twin: ``world`` virtual ranks whose
"peer-mapped" pointers are plain pointers of the same process, so every cross-GPU protocol of the suite
(step words, epochs, tickets, acks, timeouts) runs on a single-GPU box, and a single process can drive
a whole node for profiling (ncu cannot follow a multi-process launch).

One host thread enqueues for all ranks, so a kernel may only wait for work that is ALREADY enqueued
(an earlier step of a neighbour), or the waiting kernels must all be co-resident and sit on different
streams; the classes built on this (models/halo.py::VirtualRing, and ``VirtualRanks`` for the collective
miniapps) follow that rule.
"""
from __future__ import annotations

from typing import Any, List, Optional, Sequence

import torch

from .. import native
from .symmetric import SignalPads, SymmetricBuffer


class LocalComm:
    """The view one virtual rank has of its in-process group.  Barriers are no-ops (one thread drives everyone);
    scalar reductions return the rank's own value — the owner of the group aggregates."""

    backend = "local"

    def __init__(self, rank: int, world: int):
        self.rank, self.world, self.local_rank = rank, world, rank

    def barrier(self) -> None:
        pass

    def max(self, value: float) -> float:
        return float(value)

    min = max
    sum = max

    def all_gather_object(self, obj: Any) -> List[Any]:
        raise RuntimeError("LocalComm: allocate shared objects through LocalGroup")

    def close(self) -> None:
        pass


class LocalGroup:
    def __init__(self, world: int, devices: Optional[List[int]] = None):
        ndev = max(torch.cuda.device_count(), 1)
        self.world = world
        self.devices = list(devices) if devices is not None else [r % ndev for r in range(world)]
        if len(self.devices) != world:
            raise ValueError("one device per virtual rank")
        self.comms = [LocalComm(r, world) for r in range(world)]
        distinct = sorted(set(self.devices))
        if len(distinct) > 1:
            native().enable_peer_access(distinct)

    def ranks_on(self, device: int) -> int:
        return sum(1 for d in self.devices if d == device)

    def symmetric(self, nbytes: int, zero: bool = True) -> List[SymmetricBuffer]:
        return SymmetricBuffer.local_group(self.comms, nbytes, self.devices, zero)

    def pads(self, extra_words: int = 0, timeout_s: float = 20.0) -> List[SignalPads]:
        bufs = self.symmetric(SignalPads.pad_bytes(extra_words), zero=True)
        return [SignalPads(c, d, extra_words, timeout_s, buf=b) for c, d, b in zip(self.comms, self.devices, bufs)]


class VirtualRanks:
    """``world`` ranks of a collective miniapp (``models/collective.py``) driven by ONE process on one GPU: their peer
    pointers are plain pointers, and ``run_once()`` enqueues one collective per rank, each on its own stream.  Every
    rank's grid waits on its peers (per chunk, or in the node barrier it ends in), so the grids are kept co-resident:
    at most ``sms // world`` CTAs each.  At most 8 ranks: more streams than the device's hardware queues would
    serialise the spinning kernels.

    A subclass calls ``refuse``, then its own argument checks, then ``__init__``; it allocates its buffers through
    ``self.group`` and builds ``self.ranks``, one miniapp rank per virtual rank with ``ctas=self.ctas``."""

    MAX_WORLD = 8

    @classmethod
    def refuse(cls, world: int, algo: Optional[str] = None, algos: Optional[Sequence[str]] = None) -> None:
        """ValueError unless 1 <= world <= MAX_WORLD and ``algo`` is one of ``algos`` (when given)."""
        if not 1 <= world <= cls.MAX_WORLD:
            raise ValueError(f"virtual ranks: 1 <= world <= {cls.MAX_WORLD}")
        if algos is not None and algo not in algos:
            raise ValueError(f"virtual ranks run {algos}")

    def __init__(self, world: int, device: int, ctas: int):
        cap = max(1, native().sm_count(device) // world)
        self.ctas = min(ctas, cap) if ctas > 0 else cap
        self.world, self.device = world, device
        self.group = LocalGroup(world, [device] * world)
        self.streams = [torch.cuda.Stream(device) for _ in range(world)]
        self.ranks: List[Any] = []

    def run_once(self) -> None:
        """One collective: every rank's ``run_once`` on its own stream.  Call ``synchronize`` before the next one (it
        stands in for the cross-rank barrier that must separate two launches)."""
        for app, st in zip(self.ranks, self.streams):
            with torch.cuda.device(app.device), torch.cuda.stream(st):
                app.run_once()

    def synchronize(self) -> None:
        for st in self.streams:
            st.synchronize()
        for app in self.ranks:
            app.pads.check()

    def close(self) -> None:
        for app in self.ranks:
            app.close()
