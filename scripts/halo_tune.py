#!/usr/bin/env python
"""Sweep the K-halo kernel's geometry (mode x column tile x CTAs) at the benchmark's shape; one JSON row per point.

The first rows of every sweep are plain device-to-device copies of rows x bytes (torch, and the suite's ld/st and TMA
copy kernels), timed the same way: the copy ceiling of the card in that very call (a step must read and write the whole
slab, so it cannot beat that copy).

    python scripts/halo_tune.py --out gpurun_out/halo_tune.jsonl            # 1 GPU (loop-back)
    torchrun --nproc-per-node 2 scripts/halo_tune.py --out ...              # over NVLink
"""
from __future__ import annotations

import argparse
import itertools
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hpc_patterns_b200.models.halo import REFERENCE_MESSAGE_BYTES, HaloStencil  # noqa: E402
from hpc_patterns_b200.parallel.comm import Comm  # noqa: E402
from hpc_patterns_b200.utils.timing import BlockTimer  # noqa: E402


def copy_ceiling(rows: int, nbytes: int, steps: int, dev) -> list:
    """One device-to-device copy of the slab (rows x nbytes) per step, by three engines: torch's copy and the suite's
    two copy kernels (native.copy: 128-bit ld/st from every thread, and TMA bulk copies through shared memory), default
    tunings.  The engines alternate inside each of 3 blocks of `steps` copies (CUDA events); best block per engine."""
    from hpc_patterns_b200 import native

    C = native()
    n = rows * nbytes // 4
    src = torch.ones(n, dtype=torch.float32, device=dev)
    dst = torch.empty_like(src)
    st = torch.cuda.current_stream(dev).cuda_stream
    engines = {
        "d2d_copy": lambda: dst.copy_(src),
        "copy_ldst": lambda: C.copy(dst.data_ptr(), src.data_ptr(), 4 * n, False, "ldst", {}, {}, dev, st),
        "copy_tma": lambda: C.copy(dst.data_ptr(), src.data_ptr(), 4 * n, False, "tma", {}, {}, dev, st),
    }
    for run in engines.values():
        for _ in range(3):
            run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    blocks = {name: [] for name in engines}
    for _ in range(3):
        for name, run in engines.items():
            e0.record()
            for _ in range(steps):
                run()
            e1.record()
            e1.synchronize()
            blocks[name].append(round(e0.elapsed_time(e1) / steps, 5))
    del src, dst
    torch.cuda.empty_cache()
    out = []
    for name, b in blocks.items():
        ms = min(b)
        out.append({"rows": rows, "mode": name, "ms_per_step": ms, "blocks": b,
                    "hbm_GBps": round(2 * rows * nbytes / ms / 1e6, 1)})
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/halo_tune.jsonl")
    ap.add_argument("--rows", type=int, nargs="+", default=[8])
    ap.add_argument("--modes", nargs="*", default=["pull", "push"], help="none: only the copy rows")
    ap.add_argument("--tile-kb", type=int, nargs="+", default=[8, 16, 32, 64], help="column tile of a CTA in KiB")
    ap.add_argument("--ctas", type=int, nargs="+", default=[0, 132], help="0: every resident slot (2 per SM)")
    ap.add_argument("--bytes", type=int, default=REFERENCE_MESSAGE_BYTES)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--preheat-ms", type=float, default=100.0)
    args = ap.parse_args()
    comm = Comm()
    dev = comm.device
    torch.cuda.set_device(dev)
    rows_out = []
    for rows in args.rows:
        for row in copy_ceiling(rows, args.bytes, args.steps, dev):
            if comm.rank == 0:
                print(json.dumps(row), flush=True)
                rows_out.append(row)
    for rows, mode, tile_kb, ctas in itertools.product(args.rows, args.modes, args.tile_kb, args.ctas):
        tune = {"tile_kb": tile_kb}
        if ctas:
            tune["ctas"] = ctas
        try:
            hs = HaloStencil(comm, dev, args.bytes, rows, mode, tune=tune)
        except Exception as e:
            if comm.rank == 0:
                print(f"skip {mode} tile_kb={tile_kb} ctas={ctas}: {e}", flush=True)
            continue
        timer = BlockTimer(comm, hs.pads, dev)
        m = timer.measure(lambda: hs.step(args.steps), args.steps, blocks=3, preheat_ms=args.preheat_ms)
        m1 = timer.measure(lambda: [hs.step(1) for _ in range(args.steps)], args.steps, blocks=3, preheat_ms=0)
        bad = int(comm.sum(hs.verify_last_step()))
        row = {"world": comm.world, "rows": rows, "mode": mode, "tile_kb": tile_kb, "ctas": hs.ctas,
               "ms_per_step": round(m["ms"], 5), "blocks": m["blocks_ms"], "per_step_launch_ms": round(m1["ms"], 5),
               "hbm_GBps": round(hs.hbm_bytes_per_step() / m["ms"] / 1e6, 1),
               "nvlink_GBps_per_dir": round(hs.nvlink_bytes_per_step() / m["ms"] / 1e6, 1), "wrong_words": bad}
        hs.close()
        if comm.rank == 0:
            print(json.dumps(row), flush=True)
            rows_out.append(row)
    if comm.rank == 0:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "a") as f:
            for r in rows_out:
                f.write(json.dumps(r) + "\n")
    comm.close()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
