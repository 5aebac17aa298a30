"""``python -m hpc_patterns_b200 <program> [args...]`` — one front door to every pattern program.

  concurency   compute-while-copy overlap benchmark (native driver in-process)
  peer2pear    P2P bandwidth, process-per-GPU (run under torchrun for >1 GPU)
  allreduce    allreduce miniapp, process-per-GPU (run under torchrun)
  alltoall     all-to-all miniapp (push / pull kernels, nccl baseline; --counts: all-to-all-v), process-per-GPU (torchrun)
  reduce_scatter  reduce-scatter miniapp (direct kernel, nccl baseline), process-per-GPU (run under torchrun)
  allgather    all-gather miniapp (push / pull kernels, nccl baseline), process-per-GPU (run under torchrun)
  halo         the miniapp loop as a halo exchange fused into a slab stencil — the flagship (run under torchrun)
  tp           tensor-parallel linear layers with the collective fused into the GEMM, vs cuBLAS + NCCL (torchrun)
  topology     fabric planes / rank->GPU mapping (JSON)
  tile-mapping per-rank launcher: <policy> <CVD|SET> cmd...
  parse        concurrency log -> SUCCESS/FAILURE tables
  report       JSONL rows -> roofline tables
  interop      torch <-> native runtime interop demos
  build        compile the native library, CLIs and the extension in-tree
The reference's program names are accepted too: sycl_con, omp_host_threads, omp_nowait, peer2pear_i, peer2pear_w.
"""
from __future__ import annotations

import os
import sys

_GPU_PROGRAMS = ("peer2pear", "allreduce", "alltoall", "reduce_scatter", "allgather", "halo", "tp", "interop")


def _no_gpu_message(prog: str):
    """The GPU programs fail like the native CLIs on a box without a device: one line, exit status 1."""
    import torch

    if prog in _GPU_PROGRAMS and not torch.cuda.is_available():
        hint = f"; bin/{prog} --cpu is the host-only plumbing run" if prog in ("peer2pear", "allreduce", "alltoall", "reduce_scatter", "allgather") else ""
        return f"Error: {prog}: no CUDA device (this program runs sm_90a kernels{hint})"
    return None


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] in ("-h", "--help"):
        print(__doc__)
        return 0 if argv else 2
    prog, rest = argv[0], argv[1:]
    # the reference's program names
    if prog in ("sycl_con", "omp_con", "omp_host_threads", "omp_nowait"):
        rest = (["--backend", "cpu"] if prog.startswith("omp_") else []) + rest
        prog = "concurency"
    if prog in ("peer2pear_i", "peer2pear_w"):
        rest = ["--transport", "sendrecv" if prog.endswith("_i") else "put"] + rest
        prog = "peer2pear"
    if "-h" not in rest and "--help" not in rest:
        msg = _no_gpu_message(prog)
        if msg:
            print(msg, file=sys.stderr)
            return 1
    try:
        return _dispatch(prog, rest)
    except (ValueError, RuntimeError) as e:  # usage / environment problems: a message, not a traceback
        if os.environ.get("HPCP_TRACEBACK"):
            raise
        print(f"Error: {prog}: {e}", file=sys.stderr)
        return 1


def _dispatch(prog: str, rest: list) -> int:
    if prog == "concurency":
        from .models.concurency import main as m
        return m(rest)
    if prog == "peer2pear":
        from .models.peer2pear import main as m
        return m(rest)
    if prog == "allreduce":
        from .models.allreduce import main as m
        return m(rest)
    if prog == "alltoall":
        from .models.alltoall import main as m
        return m(rest)
    if prog == "reduce_scatter":
        from .models.allreduce import main_reduce_scatter as m
        return m(rest)
    if prog == "allgather":
        from .models.alltoall import main_allgather as m
        return m(rest)
    if prog == "halo":
        from .models.halo import main as m
        return m(rest)
    if prog == "tp":
        from .models.tensor_parallel import main as m
        return m(rest)
    if prog == "topology":
        from . import native
        print(native().topology_discover(rest[0] if rest else ""))
        return 0
    if prog in ("tile-mapping", "tile_mapping"):
        from .parallel.tile_mapping import main as m
        return m(rest)
    if prog == "parse":
        from .utils.parse import main as m
        return m(rest)
    if prog == "report":
        from .utils.report import main as m
        return m(rest)
    if prog == "interop":
        from .models import interop
        interop.demo_direct()
        interop.demo_native_handles()
        return 0
    if prog == "build":
        from . import _build
        _build.build(cli="--no-cli" not in rest)
        return 0
    print(f"unknown program {prog!r}\n{__doc__}", file=sys.stderr)
    return 2


if __name__ == "__main__":
    raise SystemExit(main())
