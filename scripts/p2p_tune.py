#!/usr/bin/env python
"""Sweep the K-p2p kernels' geometry at the reference's message size (one pair, torchrun --nproc-per-node 2).

One JSON row per point: transport x engine x (CTAs, stage KiB, stages | unroll, vector width, threads)."""
from __future__ import annotations

import argparse
import itertools
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hpc_patterns_b200.models.peer2pear import REFERENCE_MESSAGE_BYTES, P2PBench  # noqa: E402
from hpc_patterns_b200.parallel.comm import Comm  # noqa: E402


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/p2p_tune.jsonl")
    ap.add_argument("--bytes", type=int, default=REFERENCE_MESSAGE_BYTES)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--hybrid", action="store_true", help="only the put+get-at-once transport, over the split fraction")
    args = ap.parse_args()
    comm = Comm()
    dev = comm.device
    torch.cuda.set_device(dev)
    points = [("memcpy", "ldst", {})]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tma = [(c, kb, st) for c, kb, st in itertools.product((sms, 2 * sms, 4 * sms), (8, 16, 32, 64), (2, 4, 8))
           if kb * st <= 224 and (not args.quick or (kb, st) in ((16, 8), (32, 4), (64, 2), (8, 8)))]
    for transport in ("put", "get"):
        for c, kb, st in tma:
            points.append((transport, "tma", {"ctas": c, "stage_kb": kb, "stages": st}))
        for c, u, vec, thr in itertools.product((2 * sms, 4 * sms), (4, 8), (16, 32), (512, 1024)):
            if args.quick and not (c == 2 * sms and thr == 512):
                continue
            points.append((transport, "ldst", {"ctas": c, "unroll": u, "vec_bytes": vec, "threads": thr}))
    if args.hybrid:
        points = [("memcpy", "ldst", {})]
        for frac in (0.3, 0.4, 0.5, 0.6, 0.7):
            for engine in ("tma", "ldst"):
                points.append(("hybrid", engine, {"put_fraction": frac}))
    rows = []
    for transport, engine, tune in points:
        tune = dict(tune)
        frac = tune.pop("put_fraction", 0.5)
        try:
            b = P2PBench(comm, dev, max_bytes=args.bytes, transport=transport, engine=engine, tune=tune,
                         iters=args.iters, put_fraction=frac)
            tune["put_fraction"] = frac if transport == "hybrid" else None
            r = b.run(args.bytes, verify=True)
            b.close()
        except Exception as e:
            if comm.rank == 0:
                print(f"skip {transport} {engine} {tune}: {e!r}"[:200], flush=True)
            continue
        row = {"transport": transport, "engine": engine, **tune, "uni_GBps": round(r.uni_gbps, 1),
               "bi_GBps": round(r.bi_gbps, 1), "mismatches": r.mismatches}
        if comm.rank == 0:
            print(json.dumps(row), flush=True)
            rows.append(row)
    if comm.rank == 0:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    comm.close()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
