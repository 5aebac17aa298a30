#!/usr/bin/env python
"""All-to-all timings on one GPU with virtual ranks: bin/alltoall push, pull and --stock memcpy at 2, 4 and 8 ranks and
64 KiB, 1 MiB and 16 MiB blocks, the three variants alternated round after round in this one call, next to a torch
copy of the same P*B bytes per rank (P ranks x P*B bytes in one copy) as the HBM ceiling.  The card's name and power
limit are read in the same call.

Every rank of a virtual-rank run lives in the same HBM: these are one-HBM figures, not NVLink or NVSwitch figures.

  python scripts/alltoall_bench.py [--out rows.jsonl] [--rounds 2] [--iters 20]

Every row is printed as one JSON line; --out also writes them to a file.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = {"push": [], "pull": ["--pull"], "memcpy": ["--stock", "memcpy"]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def torch_copy_ms(nbytes, iters):
    import torch

    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(iters):
        e0.record()
        dst.copy_(src)
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    del src, dst
    torch.cuda.empty_cache()
    return best


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON rows to this file")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ranks", default="2,4,8")
    ap.add_argument("--blocks", default=f"{64 << 10},{1 << 20},{16 << 20}")
    args = ap.parse_args(argv)
    exe = os.path.join(ROOT, "bin", "alltoall")
    info = card()
    print(f"# card: {info}", flush=True)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        for rnd in range(args.rounds):
            for P in map(int, args.ranks.split(",")):
                for B in map(int, args.blocks.split(",")):
                    for variant, extra in VARIANTS.items():
                        js = os.path.join(tmp, "row.jsonl")
                        if os.path.exists(js):
                            os.remove(js)
                        p = subprocess.run([exe, "-n", str(P), "--block-bytes", str(B), "--iters", str(args.iters),
                                            "--warmup", "3", "--json", js] + extra, capture_output=True, text=True)
                        if p.returncode != 0:
                            print(p.stdout + p.stderr, file=sys.stderr)
                            return 1
                        row = json.loads(open(js).read().splitlines()[-1])
                        row.update(round=rnd, card=info)
                        rows.append(row)
                    ms = torch_copy_ms(P * P * B, args.iters)
                    rows.append({"pattern": "torch-copy", "variant": "hbm-ceiling", "ranks": P, "block_bytes": B,
                                 "bytes": P * P * B, "ms": ms, "round": rnd, "card": info})
                    line = " ".join(f"{r['variant']}={r['ms']:.4f}" for r in rows[-4:])
                    print(f"round {rnd} P={P} B={B}: {line} ms", flush=True)
    for r in rows:
        print(json.dumps(r))
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    print(f"# card: {info}", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
