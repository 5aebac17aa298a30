"""Tensor-parallel linear layers whose collective is fused into the GEMM kernel.

Beyond the reference (which has no GEMM): the suite's "compute step followed by a
collective as ONE kernel" family applied to the tensor cores.

``RowParallelLinear``     every rank holds a K-slice of the weight; ``y = reduce_scatter(x_r @ W_r.T)``.
                          One kernel: wgmma GEMM whose epilogue adds each tile into the owning rank's
                          fp32 shard over NVLink (K-gemm-rs), then a wait for the P arrival epochs.
``ColumnParallelLinear``  activations are row-sharded, the weight column-sharded:
                          ``y = all_gather(x_r) @ W_r.T``.  One kernel: gather threads pull the peers'
                          rows over NVLink while the GEMM already works on the rows that are here (K-ag-gemm).

Both keep their operands in symmetric (peer-mapped) buffers, synchronise with the suite's signal pads
(no NCCL, no host sync on the step) and carry a ``stock_forward`` that runs the same step the stock way —
``torch.matmul`` (cuBLAS) + ``torch.distributed`` reduce_scatter / all_gather (NCCL) — as the baseline.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

from .. import native
from ..ops.gemm import allgather_gemm, gemm_reduce_scatter
from ..parallel.comm import Comm
from ..parallel.symmetric import SignalPads, SymmetricBuffer


def apply_activation(y: torch.Tensor, activation: str) -> torch.Tensor:
    """Plain PyTorch form of the epilogue activations (gelu in its tanh form, like the kernel)."""
    if activation == "none":
        return y
    if activation == "relu":
        return torch.relu(y)
    if activation == "gelu":
        return torch.nn.functional.gelu(y, approximate="tanh")
    if activation == "silu":
        return torch.nn.functional.silu(y)
    raise ValueError(f"unknown activation {activation!r}")


class _FusedLinearBase:
    def __init__(self, comm: Comm, device: int, timeout_s: float):
        self.C = native()
        self.comm = comm
        self.device = device
        self.rank, self.world = comm.rank, comm.world
        self.pads = SignalPads(comm, device, timeout_s=timeout_s)
        self.epoch = 0
        self.launches = 0

    @property
    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def check(self) -> None:
        self.pads.check()


class RowParallelLinear(_FusedLinearBase):
    """``y = sum_r x_r[M, K_r] @ w_r[N, K_r].T``; ``reduce="scatter"``: every rank gets its ``[M/P, N]`` rows of the
    sum (adds into the owners' shards over NVLink); ``reduce="all"``: every rank gets the whole ``[M, N]`` sum, added
    into all copies by the NVSwitch (``multimem.red`` on the multicast mapping; needs NVLS, world >= 2)."""

    def __init__(self, comm: Comm, device: int, m: int, n: int, k_local: int, cluster: int = 0, ctas: int = 0,
                 timeout_s: float = 30.0, reduce: str = "scatter", out_dtype: torch.dtype = torch.float32,
                 epilogue: str = "red"):
        """``out_dtype=torch.bfloat16`` (reduce-scatter only): bf16 shards, half the NVLink bytes, every addition
        rounds to bf16.  ``epilogue="tma"`` (fp32 reduce-scatter): additions issued by the TMA unit (UTMAREDG)."""
        self.epilogue = epilogue
        super().__init__(comm, device, timeout_s)
        if out_dtype not in (torch.float32, torch.bfloat16) or (reduce == "all" and out_dtype != torch.float32):
            raise ValueError("out_dtype: float32, or bfloat16 with reduce='scatter'")
        self.out_dtype = out_dtype
        self.y_elem = 2 if out_dtype == torch.bfloat16 else 4
        if m % (128 * self.world) or n % 256 or k_local % 64:
            raise ValueError("M, N, K_local must be multiples of 128*world, 256, 64")
        if reduce not in ("scatter", "all"):
            raise ValueError("reduce must be 'scatter' or 'all'")
        self.m, self.n, self.k = m, n, k_local
        self.cluster, self.ctas, self.reduce = cluster, ctas, reduce
        self.w = torch.empty(n, k_local, device=f"cuda:{device}", dtype=torch.bfloat16)
        self._symm = None
        self._mc = 0
        if reduce == "all":
            import torch.distributed._symmetric_memory as symm

            try:
                if self.world < 2:
                    raise RuntimeError("reduce='all' goes through the NVSwitch multicast mapping: needs >= 2 GPUs")
                t = symm.empty(m * n, dtype=torch.float32, device=torch.device("cuda", device))
                hdl = symm.rendezvous(t, dist.group.WORLD)
                self._mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
                if self._mc == 0:
                    raise RuntimeError("torch symmetric memory reports no multicast support on this system")
            except Exception:
                self.pads.close()  # the same on every rank: nobody is left waiting in a collective
                raise
            self._symm = (t, hdl)
            self.shard = None
            self.y = t.view(m, n)
            return
        self.shard = SymmetricBuffer(comm, (m // self.world) * n * self.y_elem, device, zero=True)
        self.y = self.shard.tensor(out_dtype).view(m // self.world, n)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x: bf16 ``[M, K_local]``.  Returns this rank's rows of the reduced output (a view of the symmetric shard,
        valid until the next forward)."""
        st = self._stream
        self.epoch += 1
        self.C.memset_async(self.y.data_ptr(), 0, self.y.numel() * self.y_elem, st)
        self.pads.device_barrier(st)  # every copy / shard is zero before anybody adds into it
        done = [self.pads.word(q, self.C.PAD_DONE + self.rank) for q in range(self.world)]
        shards = self.shard.ptrs if self.shard is not None else [0] * self.world
        ctas = gemm_reduce_scatter(x, self.w, shards, self.rank, done_flags=done, done_epoch=self.epoch,
                                   ticket=self.pads.ticket_ptr, ticket_base=self.pads.ticket_issued & 0xFFFFFFFF,
                                   ctas=self.ctas, stream=st, cluster=self.cluster, c_multicast=self._mc,
                                   out_dtype=self.out_dtype, epilogue=self.epilogue)
        self.pads.advance_tickets(ctas)
        self.C.wait_flags(self.pads.word(self.rank, self.C.PAD_DONE), self.world, self.epoch, self.pads.timeout_ns,
                          self.pads.status_ptr, st)
        self.launches += 3
        return self.y

    def stock_forward(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, exact: bool = False) -> torch.Tensor:
        """cuBLAS GEMM + NCCL reduce_scatter / all_reduce (fp32), the stock pattern.  ``exact``: fp32 GEMM (the
        reference of ``--check``; the timed stock GEMM is bf16 in / bf16 out like a stock layer, whose output rounding
        is NOT what the fused layer — fp32 accumulators straight into the collective — is compared against)."""
        if x.device.type == "cpu" or exact:
            full = x.float() @ self.w.float().t()
        else:
            full = torch.matmul(x, self.w.t()).float()
        if self.world == 1:
            return full
        if self.reduce == "all":
            dist.all_reduce(full)
            return full
        out = out if out is not None else torch.empty(self.m // self.world, self.n, device=x.device)
        dist.reduce_scatter_tensor(out, full)
        return out

    def close(self) -> None:
        if self.shard is not None:
            self.shard.close()
        self._symm = None
        self.pads.close()


class ColumnParallelLinear(_FusedLinearBase):
    """``y[M, N_local] = concat_r(x_r[M/P, K]) @ w[N_local, K].T``."""

    def __init__(self, comm: Comm, device: int, m: int, n_local: int, k: int, out_dtype: torch.dtype = torch.float32,
                 cluster: int = 0, ctas: int = 0, chunk_bytes: int = 0, timeout_s: float = 30.0,
                 activation: str = "none"):
        """``activation`` (none | relu | gelu | silu) is fused into the GEMM's epilogue."""
        super().__init__(comm, device, timeout_s)
        if m % (128 * self.world) or n_local % 256 or k % 64:
            raise ValueError("M, N_local, K must be multiples of 128*world, 256, 64")
        self.activation = activation
        self.m, self.n, self.k = m, n_local, k
        self.cluster, self.ctas, self.chunk_bytes = cluster, ctas, chunk_bytes
        self.a = SymmetricBuffer(comm, m * k * 2, device, zero=True)
        self.a_full = self.a.tensor(torch.bfloat16).view(m, k)
        rows = m // self.world
        self.x_local = self.a_full[self.rank * rows:(self.rank + 1) * rows]  # write the activations here
        self.w = torch.empty(n_local, k, device=f"cuda:{device}", dtype=torch.bfloat16)
        self.y = torch.empty(m, n_local, device=f"cuda:{device}", dtype=out_dtype)
        self.ready = torch.zeros(m // 128, device=f"cuda:{device}", dtype=torch.int32)
        self.ready_base = 0
        self._per_launch = self.C.allgather_gemm_chunks_per_block(k, chunk_bytes)
        self._block_bytes = rows * k * 2

    def wait_readers(self) -> None:
        """Enqueue a wait until every peer has finished pulling this rank's rows of the previous step.  Call it
        before writing new activations into ``self.x_local`` (``forward(x_local)`` does)."""
        if self.epoch > 0 and self.world > 1:
            self.C.wait_flags(self.pads.word(self.rank, self.C.PAD_DONE), self.world, self.epoch,
                              self.pads.timeout_ns, self.pads.status_ptr, self._stream)
            self.launches += 1

    def forward(self, x_local: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x_local: this rank's bf16 rows ``[M/P, K]`` (or None when they were written into ``self.x_local``
        after ``wait_readers()``)."""
        st = self._stream
        if x_local is not None:
            self.wait_readers()
            self.x_local.copy_(x_local)
        self.pads.device_barrier(st)  # every rank's rows are final before anybody pulls them
        self.epoch += 1
        src = [self.a.ptrs[q] + q * self._block_bytes for q in range(self.world)]
        done = [self.pads.word(q, self.C.PAD_DONE + self.rank) for q in range(self.world)]
        ctas = allgather_gemm(self.a_full, src, self.w, self.y, self.rank, ready=self.ready,
                              ready_base=self.ready_base & 0xFFFFFFFF, chunk_bytes=self.chunk_bytes,
                              done_flags=done, done_epoch=self.epoch, ticket=self.pads.ticket_ptr,
                              ticket_base=self.pads.ticket_issued & 0xFFFFFFFF, timeout_ns=self.pads.timeout_ns,
                              status=self.pads.status_ptr, ctas=self.ctas, stream=st, cluster=self.cluster,
                              activation=self.activation)
        self.pads.advance_tickets(ctas)
        if self.world > 1:
            self.ready_base += self._per_launch
        self.launches += 2
        return self.y

    def stock_forward(self, x_local: torch.Tensor) -> torch.Tensor:
        """NCCL all_gather + cuBLAS GEMM (+ a separate activation kernel), the stock pattern."""
        full = x_local
        if self.world > 1:
            full = torch.empty(self.m, self.k, device=x_local.device, dtype=x_local.dtype)
            dist.all_gather_into_tensor(full, x_local.contiguous())
        return apply_activation(torch.matmul(full, self.w.t()), self.activation)

    def close(self) -> None:
        self.a.close()
        self.pads.close()


class ParallelMLP:
    """A sequence-parallel transformer MLP block on the two fused layers:

        x_rows [M/P, H]  --all-gather -> GEMM (+ activation in the epilogue)-->  h [M, F/P]
                         --GEMM -> reduce-scatter-->                             y_rows [M/P, H]

    Two kernels (plus the barrier / wait launches of the layers), no NCCL, the hidden activations h never leave the
    GPU that produced them.  ``stock_forward`` is the same block through all_gather + cuBLAS + activation kernel +
    cuBLAS + reduce_scatter."""

    def __init__(self, comm: Comm, device: int, tokens: int, hidden: int, ffn: int, activation: str = "gelu",
                 cluster: int = 0, chunk_bytes: int = 0, timeout_s: float = 30.0):
        if ffn % comm.world:
            raise ValueError("ffn must be a multiple of the world size")
        self.up = ColumnParallelLinear(comm, device, tokens, ffn // comm.world, hidden, out_dtype=torch.bfloat16,
                                       cluster=cluster, chunk_bytes=chunk_bytes, timeout_s=timeout_s,
                                       activation=activation)
        self.down = RowParallelLinear(comm, device, tokens, hidden, ffn // comm.world, cluster=cluster,
                                      timeout_s=timeout_s)

    @property
    def launches(self) -> int:
        return self.up.launches + self.down.launches

    def forward(self, x_rows: torch.Tensor) -> torch.Tensor:
        return self.down.forward(self.up.forward(x_rows))

    def stock_forward(self, x_rows: torch.Tensor) -> torch.Tensor:
        return self.down.stock_forward(self.up.stock_forward(x_rows))

    def check(self) -> None:
        self.up.check()
        self.down.check()

    def close(self) -> None:
        self.up.close()
        self.down.close()


# =====================================================================================
def _timed(fn, comm, dev, iters, warm=3):
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


def _dyadic(shape, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randint(-4, 5, shape, device=dev, generator=g).float() / 4).to(torch.bfloat16)


def main(argv: Optional[List[str]] = None) -> int:
    """``torchrun --nproc-per-node N -m hpc_patterns_b200 tp [--check] [--tokens M --out-features N --in-features K]``:
    the fused layers next to the stock pattern (cuBLAS + NCCL); one JSON line from rank 0."""
    import argparse
    import json

    ap = argparse.ArgumentParser(prog="tp")
    # Long names on purpose: under torchrun, `--m` / `--n` would be read as abbreviations of ITS options (--module,
    # --max-restarts, --nnodes, ...) even when they follow the script name.
    ap.add_argument("--tokens", dest="m", type=int, default=8192, help="M: rows (tokens) of the whole problem")
    ap.add_argument("--out-features", dest="n", type=int, default=8192, help="N: output features of the whole problem")
    ap.add_argument("--in-features", dest="k", type=int, default=8192, help="K: input features of the whole problem")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--cluster", type=int, default=0)
    ap.add_argument("--chunk", type=int, default=0, help="all-gather granularity in bytes (0 -> 4096)")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--rs-epilogue", default="red", choices=("red", "tma"),
                    help="reduce-scatter additions: REDG from the LSU, or one TMA reduce per 32x32 piece")
    ap.add_argument("--mlp", action="store_true", help="also time the two layers chained as an MLP block "
                                                       "(tokens = M, hidden = K, ffn = N)")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        print("Error: tp: no CUDA device (this program runs sm_90a kernels)", flush=True)
        return 1

    comm = Comm()
    dev = comm.device
    torch.cuda.set_device(dev)
    device = torch.device("cuda", dev)
    P = comm.world
    out = {"ranks": P, "m": args.m, "n": args.n, "k": args.k}

    # ---- row-parallel: K is sharded, the output rows are scattered -------------------------------
    k_local = args.k // P
    row = RowParallelLinear(comm, dev, args.m, args.n, k_local, cluster=args.cluster, epilogue=args.rs_epilogue)
    out["rs_epilogue"] = args.rs_epilogue
    x = _dyadic((args.m, k_local), device, 100 + comm.rank)
    row.w.copy_(_dyadic((args.n, k_local), device, 200 + comm.rank))
    if args.check:
        y = row.forward(x).clone()
        ref = row.stock_forward(x, exact=True)
        if P == 1:
            ref = ref[: args.m // P]
        torch.cuda.synchronize(dev)
        row.check()
        out["row_parallel_exact"] = bool(comm.min(float(torch.equal(y, ref))) == 1.0)
    t_fused = _timed(lambda: row.forward(x), comm, dev, args.steps)
    ref_out = torch.empty(args.m // P, args.n, device=device)
    t_stock = _timed(lambda: row.stock_forward(x, ref_out), comm, dev, args.steps)
    row.check()
    flops = 2.0 * args.m * args.n * k_local
    out["row_parallel"] = {"fused_ms": round(t_fused, 4), "stock_ms": round(t_stock, 4),
                           "speedup": round(t_stock / t_fused, 3),
                           "fused_tflops_per_gpu": round(flops / t_fused / 1e9, 1),
                           "nvlink_GBps_per_gpu": round(args.m * args.n * 4 * (P - 1) / P / (t_fused * 1e6), 1)}
    row.close()

    # ---- row-parallel with an all-reduce through the switch (NVLS) -------------------------------
    if P > 1:
        try:
            ar = RowParallelLinear(comm, dev, args.m, args.n, k_local, cluster=args.cluster, reduce="all")
        except RuntimeError as e:  # no multicast support on this system
            ar = None
            out["row_parallel_allreduce"] = {"unavailable": str(e)[:120]}
        if ar is not None:
            ar.w.copy_(_dyadic((args.n, k_local), device, 200 + comm.rank))
            if args.check:
                y = ar.forward(x).clone()
                ref = ar.stock_forward(x, exact=True)
                torch.cuda.synchronize(dev)
                ar.check()
                out["row_parallel_allreduce_exact"] = bool(comm.min(float(torch.equal(y, ref))) == 1.0)
            t_fused = _timed(lambda: ar.forward(x), comm, dev, args.steps)
            t_stock = _timed(lambda: ar.stock_forward(x), comm, dev, args.steps)
            ar.check()
            out["row_parallel_allreduce"] = {"fused_ms": round(t_fused, 4), "stock_ms": round(t_stock, 4),
                                             "speedup": round(t_stock / t_fused, 3),
                                             "nvlink_out_GBps_per_gpu": round(args.m * args.n * 4 / (t_fused * 1e6), 1)}
            ar.close()

    # ---- column-parallel: rows of x are sharded and gathered, N is sharded -------------------------
    n_local = args.n // P
    col = ColumnParallelLinear(comm, dev, args.m, n_local, args.k, out_dtype=torch.bfloat16, cluster=args.cluster,
                               chunk_bytes=args.chunk)
    x_rows = _dyadic((args.m // P, args.k), device, 300 + comm.rank)
    col.w.copy_(_dyadic((n_local, args.k), device, 400 + comm.rank))
    if args.check:
        y = col.forward(x_rows).clone()
        ref = col.stock_forward(x_rows)
        torch.cuda.synchronize(dev)
        col.check()
        out["column_parallel_exact"] = bool(comm.min(float(torch.equal(y, ref.to(y.dtype)))) == 1.0)
    t_fused = _timed(lambda: col.forward(x_rows), comm, dev, args.steps)
    t_stock = _timed(lambda: col.stock_forward(x_rows), comm, dev, args.steps)
    col.check()
    flops = 2.0 * args.m * n_local * args.k
    out["column_parallel"] = {"fused_ms": round(t_fused, 4), "stock_ms": round(t_stock, 4),
                              "speedup": round(t_stock / t_fused, 3),
                              "fused_tflops_per_gpu": round(flops / t_fused / 1e9, 1),
                              "nvlink_GBps_per_gpu": round(args.m * args.k * 2 * (P - 1) / P / (t_fused * 1e6), 1)}
    col.close()

    # ---- the two layers as one MLP block (activation fused into the first GEMM's epilogue) -------------
    if args.mlp:
        mlp = ParallelMLP(comm, dev, args.m, args.k, args.n, activation="relu" if args.check else "gelu",
                          cluster=args.cluster, chunk_bytes=args.chunk)       # hidden = K, ffn = N
        mlp.up.w.copy_(_dyadic((args.n // P, args.k), device, 500 + comm.rank) / 8)
        mlp.down.w.copy_(_dyadic((args.k, args.n // P), device, 600 + comm.rank))
        xr = _dyadic((args.m // P, args.k), device, 700 + comm.rank)
        if args.check:
            y = mlp.forward(xr).clone()
            ref = mlp.stock_forward(xr)
            if P == 1:
                ref = ref[: args.m]
            torch.cuda.synchronize(dev)
            mlp.check()
            out["mlp_max_abs_diff"] = comm.max(float((y - ref).abs().max()))
            out["mlp_ref_max_abs"] = comm.max(float(ref.abs().max()))
        t_fused = _timed(lambda: mlp.forward(xr), comm, dev, args.steps)
        t_stock = _timed(lambda: mlp.stock_forward(xr), comm, dev, args.steps)
        mlp.check()
        out["mlp"] = {"fused_ms": round(t_fused, 4), "stock_ms": round(t_stock, 4),
                      "speedup": round(t_stock / t_fused, 3),
                      "fused_tflops_per_gpu": round(4.0 * args.m * (args.n // P) * args.k / t_fused / 1e9, 1)}
        mlp.close()
    if comm.rank == 0:
        print(json.dumps(out), flush=True)
    ok = (not args.check) or (out["row_parallel_exact"] and out["column_parallel_exact"] and
                              out.get("row_parallel_allreduce_exact", True))
    comm.close()
    return 0 if ok else 1

