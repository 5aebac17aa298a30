#!/usr/bin/env python
"""K-halo by field type on one GPU: float, double, bfloat16 and half, pull mode, N = 1, 8 rows.

Two sets of cases:
  * equal bytes: every type at the benchmark's row of 188 743 680 B (what bench.py runs for float);
  * equal elements: double, bfloat16 and half at float's 47 185 920 elements per row.
The cases alternate inside each of three rounds.  A case is timed with BlockTimer (best of 5 blocks of 20 steps, one
persistent launch per block) next to a torch copy of its slab (best of 5 blocks of 20 copies, CUDA events), and its last
step is checked exactly (verify_last_step).  HBM GB/s is 2 * rows * row_bytes / t, the bytes a step must move.  The card
name and power limit are read in the same call.

    python scripts/halo_dtype_bench.py [--out rows.jsonl]      # --out: also append the JSON rows to a file
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hpc_patterns_b200.models.halo import DTYPES, REFERENCE_MESSAGE_BYTES, HaloStencil  # noqa: E402
from hpc_patterns_b200.parallel.comm import Comm  # noqa: E402
from hpc_patterns_b200.utils.timing import BlockTimer  # noqa: E402


def card(dev: int) -> dict:
    q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def copy_ms(nbytes: int, steps: int, blocks: int, dev: int) -> tuple:
    """A torch device-to-device copy of the slab: best and all of `blocks` blocks of `steps` copies, ms per copy."""
    src = torch.ones(nbytes // 4, dtype=torch.float32, device=dev)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(blocks):
        e0.record()
        for _ in range(steps):
            dst.copy_(src)
        e1.record()
        e1.synchronize()
        out.append(round(e0.elapsed_time(e1) / steps, 5))
    del src, dst
    return min(out), out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="append the JSON rows to this file")
    ap.add_argument("--rows", type=int, default=8)
    ap.add_argument("--bytes", type=int, default=REFERENCE_MESSAGE_BYTES)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    comm = Comm()
    if comm.world != 1:
        raise SystemExit("halo_dtype_bench runs on one GPU (N = 1)")
    dev = comm.device
    torch.cuda.set_device(dev)
    info = card(dev)
    print(json.dumps(info), flush=True)
    elems = args.bytes // 4
    cases = [("equal_bytes", dt, args.bytes) for dt in DTYPES]
    cases += [("equal_elems", dt, elems * torch.empty(0, dtype=dt).element_size()) for dt in DTYPES
              if dt != torch.float32]
    ring = {c: HaloStencil(comm, dev, c[2], args.rows, "pull", dtype=c[1]) for c in cases}
    timer = BlockTimer(comm, ring[cases[0]].pads, dev)
    rows = []
    for rnd in range(args.rounds):
        for c in cases:
            hs = ring[c]
            timer.pads = hs.pads
            m = timer.measure(lambda: hs.step(args.steps), args.steps, blocks=args.blocks, preheat_ms=100.0)
            cms, cblocks = copy_ms(args.rows * c[2], args.steps, args.blocks, dev)
            row = {"round": rnd, "set": c[0], "type": DTYPES[c[1]], "rows": args.rows, "row_bytes": c[2],
                   "row_elems": hs.row_elems, "ms_per_step": round(m["ms"], 5), "blocks_ms": m["blocks_ms"],
                   "spread_pct": m["spread_pct"], "hbm_GBps": round(2 * args.rows * c[2] / m["ms"] / 1e6, 1),
                   "torch_copy_ms": cms, "torch_copy_GBps": round(2 * args.rows * c[2] / cms / 1e6, 1),
                   "torch_copy_blocks_ms": cblocks, "wrong_words": hs.verify_last_step(), **info}
            print(json.dumps(row), flush=True)
            rows.append(row)
    print("\n| set | type | ms/step (min-max over rounds) | HBM GB/s | torch copy GB/s | spread % | wrong |")
    print("|---|---|---|---|---|---|---|")
    for c in cases:
        rs = [r for r in rows if r["set"] == c[0] and r["type"] == DTYPES[c[1]]]
        t = [r["ms_per_step"] for r in rs]
        print(f"| {c[0]} | {DTYPES[c[1]]} | {min(t):.3f}-{max(t):.3f} | "
              f"{min(r['hbm_GBps'] for r in rs):.0f}-{max(r['hbm_GBps'] for r in rs):.0f} | "
              f"{min(r['torch_copy_GBps'] for r in rs):.0f}-{max(r['torch_copy_GBps'] for r in rs):.0f} | "
              f"{min(r['spread_pct'] for r in rs):.2f}-{max(r['spread_pct'] for r in rs):.2f} | "
              f"{sum(r['wrong_words'] for r in rs)} |", flush=True)
    for hs in ring.values():
        hs.close()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    comm.close()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
