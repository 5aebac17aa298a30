#!/usr/bin/env bash
# maxloc / minloc against max of the same bytes per element, four virtual ranks on one GPU, two rounds that alternate
# the ops: float_int (8 bytes) against long at -p 25, double_int (16 bytes) at -p 24 against long at -p 25.
# Usage: scripts/loc_bench.sh [OUT.jsonl]  (the card's name and power limit are printed first)
set -euo pipefail
cd "$(dirname "$0")/.."
out=${1:-loc_bench.jsonl}
nvidia-smi --query-gpu=name,power.limit --format=csv,noheader
for round in 1 2; do
  for algo in "--algo ring" "--algo ring-rsag" "-a"; do
    bin/allreduce.long -n 4 -p 25 --iters 5 --op max $algo --json "$out" | grep Elapsed
    bin/allreduce.float_int -n 4 -p 25 --iters 5 --op maxloc $algo --json "$out" | grep Elapsed
    bin/allreduce.float_int -n 4 -p 25 --iters 5 --op minloc $algo --json "$out" | grep Elapsed
    bin/allreduce.double_int -n 4 -p 24 --iters 5 --op maxloc $algo --json "$out" | grep Elapsed
    bin/allreduce.double_int -n 4 -p 24 --iters 5 --op minloc $algo --json "$out" | grep Elapsed
  done
done
