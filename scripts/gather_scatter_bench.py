#!/usr/bin/env python
"""Reduce-scatter and all-gather timings on one GPU with virtual ranks, every arm alternated round after round in this
one call; the card's name and power limit are read in the same call.

  reduce-scatter (float sum and bfloat16 sum, segments of S bytes):
      direct      the one-launch reduce-scatter (VirtualReduceScatter)
      ring-rs     the reduce-scatter phase of the ring-rsag kernel (native().ring_rsag(..., phases="reduce_scatter"))
  all-gather (blocks of S bytes):
      push, pull  the one-launch all-gather (VirtualAllgather)
      memcpy      the stock shape of `bin/allgather --stock memcpy`: P-1 peer copies plus the local one per rank
                  (cudaMemcpyAsync through torch's copy_) in the staggered order, then the device barrier
      ring-ag     the all-gather phase of the ring-rsag kernel (phases="all_gather")
  hbm-ceiling     a torch copy of P*P*S bytes: what all ranks' receive buffers get in an all-gather, and what all ranks
                  load in a reduce-scatter

A time is the least over --iters launches of (the last rank's end - the common start), with CUDA events.  Every rank of
a virtual-rank run lives in the same HBM: these are one-HBM figures, not NVLink or NVSwitch figures.

  python scripts/gather_scatter_bench.py [--out rows.jsonl] [--rounds 2] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(streams, launch, iters, between):
    """Least over iters of the time from a common start to the last rank's end; ``launch(r)`` enqueues rank r."""
    import torch

    best = float("inf")
    for it in range(iters + 3):
        start = torch.cuda.Event(enable_timing=True)
        ends = [torch.cuda.Event(enable_timing=True) for _ in streams]
        start.record(streams[0])
        for st in streams[1:]:
            st.wait_event(start)
        for r, st in enumerate(streams):
            with torch.cuda.stream(st):
                launch(r)
            ends[r].record(st)
        for st in streams:
            st.synchronize()
        between()
        if it >= 3:
            best = min(best, max(start.elapsed_time(e) for e in ends))
    return best


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


def ring_phase(P, seg_bytes, dtype, phase, iters):
    """One phase of the ring-rsag kernel on P virtual ranks, segments of seg_bytes."""
    from hpc_patterns_b200 import native
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    C = native()
    esz = C.elem_size(dtype)
    v = VirtualAllreduce(P, P * seg_bytes // esz, dtype, "ring-rsag")
    code = C.RSAG_REDUCE_SCATTER if phase == "reduce_scatter" else C.RSAG_ALL_GATHER
    try:
        def launch(r):
            app = v.ranks[r]
            pads, me, right = app.pads, app.rank, app.right
            C.ring_rsag(va=app.va.local_ptr, vc=app.vc.local_ptr, slots_local=app.slots.local_ptr,
                        slots_right=app.slots.ptrs[right], vc_right=app.vc.ptrs[right],
                        arrived_local=pads.chunk_word(me), arrived_right=pads.chunk_word(right), rank=me, world=P,
                        n=app.n, chunk_elems=0, epoch_base=app.ring_epoch, timeout_ns=pads.timeout_ns,
                        status=pads.status_ptr, dtype=dtype, ctas=v.ctas, device=0,
                        stream=__import__("torch").cuda.current_stream().cuda_stream, phases=phase)
            app.ring_epoch += C.rsag_epoch_advance(code, P)

        return timed(v.streams, launch, iters, v.synchronize)
    finally:
        v.close()


def main(argv):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON rows to this file")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ranks", default="2,4,8")
    ap.add_argument("--sizes", default=f"{64 << 10},{1 << 20},{16 << 20}")
    args = ap.parse_args(argv)
    import torch

    import hpc_patterns_b200  # noqa: F401  (before CUDA starts: eager module loading)
    from hpc_patterns_b200.models.allreduce import VirtualReduceScatter
    from hpc_patterns_b200.models.alltoall import VirtualAllgather

    info = card()
    print(f"# card: {info}", flush=True)
    rows = []
    for rnd in range(args.rounds):
        for P in map(int, args.ranks.split(",")):
            for S in map(int, args.sizes.split(",")):
                here = []
                for dtype in ("float", "bfloat16"):
                    esz = 4 if dtype == "float" else 2
                    v = VirtualReduceScatter(P, S // esz, dtype, "sum")
                    ms = timed(v.streams, lambda r: v.ranks[r].run_once(), args.iters, v.synchronize)
                    v.close()
                    here.append({"pattern": "reduce_scatter", "variant": "direct", "type": dtype, "ms": ms})
                    here.append({"pattern": "reduce_scatter", "variant": "ring-rs", "type": dtype,
                                 "ms": ring_phase(P, S, dtype, "reduce_scatter", args.iters)})
                for algo in ("push", "pull"):
                    v = VirtualAllgather(P, S, algo)
                    ms = timed(v.streams, lambda r: v.ranks[r].run_once(), args.iters, v.synchronize)
                    v.close()
                    here.append({"pattern": "allgather", "variant": algo, "ms": ms})
                v = VirtualAllgather(P, S, "push")

                def memcpy_shape(r, v=v, P=P, S=S):
                    src = v.ranks[r].send.tensor()
                    for j in range(P):
                        p = (r + 1 + j) % P
                        v.ranks[p].recv.tensor()[r * S:(r + 1) * S].copy_(src)
                    v.ranks[r].pads.device_barrier(torch.cuda.current_stream().cuda_stream)

                ms = timed(v.streams, memcpy_shape, args.iters, v.synchronize)
                v.close()
                here.append({"pattern": "allgather", "variant": "memcpy", "ms": ms})
                here.append({"pattern": "allgather", "variant": "ring-ag",
                             "ms": ring_phase(P, S, "float", "all_gather", args.iters)})
                here.append({"pattern": "torch-copy", "variant": "hbm-ceiling", "bytes": P * P * S,
                             "ms": torch_copy_ms(P * P * S, args.iters)})
                for row in here:
                    row.update(ranks=P, segment_bytes=S, round=rnd, card=info)
                    if row["pattern"] != "torch-copy":
                        row["GBps_sent_per_rank"] = (P - 1) * S / (row["ms"] * 1e-3) / 1e9
                rows += here
                line = " ".join(f"{r['pattern'][:2]}-{r['variant']}{'-' + r['type'] if 'type' in r else ''}"
                                f"={r['ms']:.4f}" for r in here)
                print(f"round {rnd} P={P} S={S}: {line} ms", flush=True)
                torch.cuda.empty_cache()
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
