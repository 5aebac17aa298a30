"""What the per-rank collective miniapps share (``models/allreduce.py``, ``models/alltoall.py``): the rank plumbing, the
timed and checked loop of ``run()`` and the CLI's report.

A collective's Python twin subclasses ``CollectiveMiniapp`` and supplies ``initialize`` (the constant or seeded data of
one iteration), ``run_once`` (enqueue one collective on the current stream), ``mismatches`` (this rank's wrong
elements or words after the last iteration) and ``result`` (the JSON-row dataclass); its virtual-rank driver subclasses
``parallel.local.VirtualRanks``, and its CLI main ends in ``report``.
"""
from __future__ import annotations

import json
from typing import Optional, Sequence

import torch

from ..parallel.comm import Comm
from ..utils.timing import BlockTimer


def gbps(sent_bytes: float, ms: float) -> float:
    """GB/s of ``sent_bytes`` in ``ms`` milliseconds (0 for an untimed result)."""
    return sent_bytes / (ms * 1e-3) / 1e9 if ms > 0 else 0.0


class CollectiveMiniapp:
    """One rank of a collective miniapp.  ``PATTERN`` names it in NVTX ranges, ``UNIT`` is what ``mismatches`` counts,
    ``BUFFERS`` are the attributes holding the symmetric buffers the rank closes (``None`` when an algorithm has none)."""

    PATTERN = ""
    UNIT = "words"
    BUFFERS: Sequence[str] = ("send", "recv")

    def __init__(self, comm: Comm, device: int, C, algo: str, ctas: int, shared: Optional[dict],
                 virtual_algos: Sequence[str]):
        """Call after the subclass's own refusals.  ``C`` is the native extension as the subclass's module resolves it
        (``native()`` there, which the emulated device of the CPU tests replaces); ``shared`` is the ``_shared``
        buffers of a virtual rank, which only the ``virtual_algos`` can use."""
        if shared is not None and algo not in virtual_algos:
            names = virtual_algos[0] if len(virtual_algos) == 1 else virtual_algos
            raise ValueError(f"virtual ranks run {names}: {algo} needs one process per GPU")
        self.C = C
        self.comm, self.device = comm, device
        self.rank, self.world = comm.rank, comm.world
        self.algo, self.ctas = algo, ctas
        self.launch_ctas = 0
        torch.cuda.set_device(device)

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def at_best(self) -> None:
        """Called by ``run()`` after the fastest timed iteration so far: state the result reports beside its time."""

    def run(self, iters: int = 5, warmup: int = 1, *init_args):
        """``warmup + iters`` iterations of ``initialize(*init_args)`` and one timed ``run_once`` (``BlockTimer``: the
        device barrier right before the start event, max over ranks), then this rank's check and its verdict line.
        The result holds the least timed iteration and the mismatches summed over ranks.  Each iteration is one NVTX
        range, ``"<PATTERN> <algo> warm-up|timed"``; nothing but ``run_once`` runs between the two events."""
        timer = BlockTimer(self.comm, self.pads, self.device)
        best = float("inf")
        for it in range(warmup + iters):
            with torch.cuda.nvtx.range(f"{self.PATTERN} {self.algo} {'warm-up' if it < warmup else 'timed'}"):
                self.initialize(*init_args)
                t = timer.block_ms(self.run_once)
            if it >= warmup and t < best:
                best = t
                self.at_best()
        bad = self.mismatches()
        total_bad = int(self.comm.sum(bad))
        print(f"Passed {self.rank}" if bad == 0 else f"FAILED {self.rank}: {bad} wrong {self.UNIT}", flush=True)
        return self.result(best, total_bad)

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        for name in self.BUFFERS:
            buf = getattr(self, name)
            if buf is not None:
                buf.close()
        self.pads.close()


def report(comm: Comm, app: CollectiveMiniapp, res, args, what: str) -> int:
    """The end of a CLI main: rank 0 prints the time, ``what`` ran and the GB/s, and appends the JSON row to
    ``args.json``; then the rank and the communicator are closed.  The exit code is 1 if any rank saw a mismatch."""
    if comm.rank == 0:
        row = res.row()
        print(f"Elapsed (max over ranks, min of {args.iters}): {res.ms:.4f} ms | {what} | "
              f"{row['GBps_sent_per_rank']:.1f} GB/s sent per rank", flush=True)
        if args.json:
            with open(args.json, "a") as f:
                f.write(json.dumps(row) + "\n")
    app.close()
    comm.close()
    return 0 if res.mismatches == 0 else 1
