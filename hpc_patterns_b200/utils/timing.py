"""Device timing helpers: CUDA events on the launching stream, max over ranks, min over blocks.

The reference times on the host and reports the minimum over 10 iterations of
"max over ranks of end - min over ranks of start" (p2p/peer2pear.cpp:23,46-52).  Here a timed block is
bracketed on the device: an in-kernel cross-GPU barrier is the last thing enqueued before the start
event on every rank, so host-side skew between ranks (a slow NVML call, a late Python thread) cannot
leak into the region; the block's time is the max over ranks of the event interval, a measurement is
the min over several blocks, and every series starts with a time-based pre-heat so a GPU that just left
idle clocks is not what gets reported.
"""
from __future__ import annotations

import statistics
import time
from typing import Callable, Dict, List, Optional

import torch


def time_region_ms(fn: Callable[[], None], device: int, stream: torch.cuda.Stream | None = None) -> float:
    """Elapsed device milliseconds of everything ``fn`` enqueues on the current stream (single rank)."""
    stream = stream or torch.cuda.current_stream(device)
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(device)
    e0.record(stream)
    fn()
    e1.record(stream)
    torch.cuda.synchronize(device)
    return float(e0.elapsed_time(e1))


def flush_l2(device: int, nbytes: int = 256 << 20) -> None:
    """Evict L2 (50 MB on H100) by writing a larger scratch buffer."""
    buf = getattr(flush_l2, "_buf", None)
    if buf is None or buf.numel() < nbytes or buf.device.index != device:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=torch.device("cuda", device))
        flush_l2._buf = buf
    buf.fill_(1)


class BlockTimer:
    """Times blocks of work that every rank enqueues: barrier + synchronize on both sides, an in-kernel
    cross-GPU barrier right before the start event, CUDA events on the launching stream, max over ranks."""

    def __init__(self, comm, pads, device: int):
        self.comm, self.pads, self.device = comm, pads, device
        self.stream = torch.cuda.current_stream(device)

    def block_ms(self, enqueue: Callable[[], None], after: Optional[Callable[[], None]] = None) -> float:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(self.device)
        self.comm.barrier()
        self.pads.device_barrier(self.stream.cuda_stream)   # the region starts behind a device-side barrier
        e0.record(self.stream)
        enqueue()
        e1.record(self.stream)
        torch.cuda.synchronize(self.device)
        self.comm.barrier()
        if after is not None:
            after()
        self.pads.check()
        return float(self.comm.max(e0.elapsed_time(e1)))

    def preheat(self, enqueue: Callable[[], None], min_ms: float) -> Dict:
        """Run ``enqueue`` blocks until at least ``min_ms`` of device time was spent — the same count on every rank
        (the count is agreed from the first block's time, never from a per-rank clock)."""
        t_first = self.block_ms(enqueue)
        reps = 0
        if min_ms > t_first:
            reps = int(self.comm.max((min_ms - t_first) / max(t_first, 1e-3))) + 1
        t0 = time.perf_counter()
        for _ in range(reps):
            enqueue()
        torch.cuda.synchronize(self.device)
        self.comm.barrier()
        self.pads.check()
        return {"blocks": reps + 1, "ms": round(t_first + (time.perf_counter() - t0) * 1e3, 1)}

    def measure(self, enqueue: Callable[[], None], units: int, blocks: int = 5, preheat_ms: float = 300.0,
                warmup: Optional[Callable[[], None]] = None) -> Dict:
        """min / median / max of ``blocks`` timed blocks, each ``units`` steps, in ms per step."""
        heat = self.preheat(enqueue, preheat_ms) if preheat_ms > 0 else {"blocks": 0, "ms": 0.0}
        if warmup is not None:
            warmup()
        per: List[float] = [self.block_ms(enqueue) / units for _ in range(blocks)]
        return {"ms": min(per), "median_ms": statistics.median(per), "max_ms": max(per),
                "blocks_ms": [round(x, 5) for x in per], "preheat_ms": heat["ms"],
                "spread_pct": round(100.0 * (max(per) - min(per)) / min(per), 2)}
