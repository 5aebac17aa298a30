#!/usr/bin/env python
"""K-gemm-put vs the stock pattern (cuBLAS matmul, then a copy-engine peer copy).

1 GPU : GEMM-only throughput of the hand-written wgmma kernel next to torch.matmul (cuBLAS).
N GPUs: (torchrun) every rank computes C = A.B^T and puts it into its ring neighbour —
        fused in the kernel's epilogue vs matmul + cudaMemcpyAsync to the peer mapping.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hpc_patterns_b200.ops.gemm import gemm_put  # noqa: E402
from hpc_patterns_b200.parallel.comm import Comm  # noqa: E402
from hpc_patterns_b200.parallel.symmetric import SignalPads, SymmetricBuffer  # noqa: E402
from hpc_patterns_b200 import native  # noqa: E402


def timed(fn, comm, dev, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(dev)
    best = float("inf")
    for _ in range(iters):
        comm.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(dev)
        best = min(best, comm.max(e0.elapsed_time(e1)))
    return best


def main():
    comm = Comm()
    dev = comm.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    C = native()
    shapes = [(8192, 8192, 1024), (8192, 8192, 2048), (8192, 8192, 4096), (8192, 8192, 8192)]
    right, left = (comm.rank + 1) % comm.world, (comm.rank - 1) % comm.world
    pads = SignalPads(comm, dev)
    rows = []
    for m, n, k in shapes:
        a = torch.randn(m, k, device=f"cuda:{dev}").to(torch.bfloat16)
        b = torch.randn(n, k, device=f"cuda:{dev}").to(torch.bfloat16)
        c = torch.empty(m, n, device=f"cuda:{dev}", dtype=torch.bfloat16)
        recv = SymmetricBuffer(comm, m * n * 2, dev, zero=False)
        flops = 2.0 * m * n * k
        st = lambda: torch.cuda.current_stream(dev).cuda_stream  # noqa: E731
        t_single = timed(lambda: gemm_put(a, b, c, 0, out_dtype=torch.bfloat16, cluster=1), comm, dev)
        t_ours = timed(lambda: gemm_put(a, b, c, 0, out_dtype=torch.bfloat16), comm, dev)
        c_ref = torch.empty(m, n, device=f"cuda:{dev}", dtype=torch.bfloat16)
        t_cublas = timed(lambda: torch.matmul(a, b.t(), out=c_ref), comm, dev)
        row = {"m": m, "n": n, "k": k, "ranks": comm.world, "out": "bf16", "gemm_ms": t_ours,
               "gemm_tflops": flops / t_ours / 1e9, "gemm_tflops_no_cluster": flops / t_single / 1e9,
               "cublas_ms": t_cublas, "cublas_tflops": flops / t_cublas / 1e9,
               "max_abs_diff_vs_cublas": float((c.float() - c_ref.float()).abs().max())}
        if True:  # TMA-store epilogue (UTMASTG)
            t_tma = timed(lambda: gemm_put(a, b, c, 0, out_dtype=torch.bfloat16, epilogue="tma"), comm, dev)
            row["gemm_tflops_tma_epilogue"] = flops / t_tma / 1e9
            row["max_abs_diff_tma_epilogue_vs_cublas"] = float((c.float() - c_ref.float()).abs().max())
        epoch = [0]

        def fused():
            epoch[0] += 1
            sync = pads.sync_ops(signal_rank=right, signal_section=C.PAD_DONE, epoch=epoch[0])
            pads.advance_tickets(gemm_put(a, b, None, recv.ptrs[right], sync=sync, out_dtype=torch.bfloat16))
            C.wait(pads.word(comm.rank, C.PAD_DONE + left), epoch[0], pads.timeout_ns, pads.status_ptr, st())

        def stock():
            torch.matmul(a, b.t(), out=c_ref)                                  # cuBLAS bf16 GEMM
            C.memcpy_async(recv.ptrs[right], c_ref.data_ptr(), m * n * 2, st())  # copy-engine put

        row["fused_gemm_put_ms"] = timed(fused, comm, dev)
        row["stock_cublas_then_memcpy_ms"] = timed(stock, comm, dev)
        row["speedup_vs_stock"] = row["stock_cublas_then_memcpy_ms"] / row["fused_gemm_put_ms"]
        pads.check()
        rows.append(row)
        if comm.rank == 0:
            print(json.dumps(row), flush=True)
        recv.close()
    pads.close()
    comm.close()


if __name__ == "__main__":
    main()
