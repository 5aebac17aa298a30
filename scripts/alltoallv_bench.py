#!/usr/bin/env python
"""All-to-all-v timings on one GPU with virtual ranks, at 2, 4 and 8 ranks and mean segments of 64 KiB, 1 MiB and
16 MiB (rows of 4 KiB), every arm alternated round after round in this one call:

  block        the equal-block kernel (bin/alltoall) at the same bytes: the yardstick of the v kernel at equal counts
  v-equal      the all-to-all-v kernel with every count the mean (--counts equal): the cost of reading the count matrix
               and of the variable walk
  v-random     --counts random, push and pull
  v-skewed     --counts skewed: one hot receiver takes most of the rows
  v-memcpy     --counts random --stock memcpy: P cudaMemcpyAsync at host-known displacements, what a design that
               synchronised the host for the counts gets after paying for that sync
  torch-copy   one torch copy of P*P*B bytes, the HBM ceiling

The card's name and power limit are read in the same call.  Every rank of a virtual-rank run lives in the same HBM:
these are one-HBM figures, not NVLink or NVSwitch figures.

  python scripts/alltoallv_bench.py [--out rows.jsonl] [--rounds 2] [--iters 20]

Every row is printed as one JSON line; --out also writes them to a file.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from alltoall_bench import card, torch_copy_ms  # noqa: E402

ROW_BYTES = 4096
ARMS = {"block": [], "v-equal": ["--counts", "equal"], "v-random": ["--counts", "random"],
        "v-random-pull": ["--counts", "random", "--pull"], "v-skewed": ["--counts", "skewed"],
        "v-memcpy": ["--counts", "random", "--stock", "memcpy"]}


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
                    for arm, extra in ARMS.items():
                        js = os.path.join(tmp, "row.jsonl")
                        if os.path.exists(js):
                            os.remove(js)
                        rb = ["--row-bytes", str(ROW_BYTES)] if extra else []
                        p = subprocess.run([exe, "-n", str(P), "--block-bytes", str(B), "--iters", str(args.iters),
                                            "--warmup", "3", "--json", js] + extra + rb, capture_output=True, text=True)
                        if p.returncode != 0:
                            print(p.stdout + p.stderr, file=sys.stderr)
                            return 1
                        row = json.loads(open(js).read().splitlines()[-1])
                        row.update(arm=arm, round=rnd, card=info)
                        rows.append(row)
                    ms = torch_copy_ms(P * P * B, args.iters)
                    rows.append({"pattern": "torch-copy", "arm": "torch-copy", "ranks": P, "block_bytes": B,
                                 "bytes": P * P * B, "ms": ms, "round": rnd, "card": info})
                    line = " ".join(f"{r['arm']}={r['ms']:.4f}" for r in rows[-len(ARMS) - 1:])
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
