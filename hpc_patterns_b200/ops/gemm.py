"""K-gemm-put: wgmma bf16 GEMM whose epilogue stores the result tile into a peer GPU.

``gemm_put(a, b, c_local=..., c_peer=...)`` computes ``C = A @ B.T`` (A ``[M,K]``, B ``[N,K]``, both
bf16 row-major, fp32 result) with the hand-written sm_90a kernel in ``csrc/kernels/gemm_put.cu``
(TMA-fed smem ring, ``wgmma.mma_async`` accumulating in registers, epilogue straight from the registers) and writes every
128x256 tile to ``c_local`` and/or straight into the peer-mapped ``c_peer`` over NVLink.
The reference has no GEMM; this op is the tensor-core member of the suite's fused
"produce a tile -> put it to the neighbour" family.  Stock comparison: ``torch.matmul`` (cuBLAS)
followed by a copy-engine peer copy.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from .. import native
from ._util import PtrLike, current_stream, ptr


def gemm_put(a: torch.Tensor, b: torch.Tensor, c_local: Optional[torch.Tensor] = None, c_peer: PtrLike = 0,
             sync: Optional[dict] = None, ctas: int = 0, stream: Optional[int] = None,
             out_dtype: torch.dtype = torch.float32, cluster: int = 0, epilogue: str = "st") -> int:
    """Launch the fused GEMM(+put).  ``out_dtype`` fp32 or bf16 (c_local / c_peer hold that type).
    ``cluster``: 0 auto, 1 = single CTAs, 2 = CTA pairs sharing the B tile through TMA multicast.
    ``epilogue``: ``"st"`` = 128-bit stores from the consumer warps, ``"tma"`` (opt-in) = swizzled smem pieces +
    ``cp.async.bulk.tensor.2d`` stores issued by the TMA unit.
    fp32 results below 2^-126 (subnormal) are kept exactly by both epilogues: the tensor cores do not flush them
    (measured on an H100, tests/test_gpu_gemm_numerics.py).  bf16 output is the fp32 accumulator rounded to nearest even.
    Returns the number of CTAs launched (for ticket bookkeeping)."""
    if epilogue not in ("st", "tma"):
        raise ValueError("epilogue must be 'st' or 'tma'")
    if out_dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("out_dtype must be float32 or bfloat16")
    if a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise TypeError("gemm_put takes bf16 operands")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[1]:
        raise ValueError("expected A[M,K] and B[N,K]")
    m, k = a.shape
    n = b.shape[0]
    if m % 128 or n % 256 or k % 64:
        raise ValueError("M, N, K must be multiples of 128, 256, 64")
    if c_local is not None and (c_local.dtype != out_dtype or tuple(c_local.shape) != (m, n)):
        raise ValueError("c_local must be [M,N] of out_dtype")
    if isinstance(c_peer, torch.Tensor) and (c_peer.dtype != out_dtype or tuple(c_peer.shape) != (m, n)):
        raise ValueError("c_peer must be [M,N] of out_dtype")
    dev = a.device.index
    return native().gemm_put(ptr(a), ptr(b), ptr(c_local) if c_local is not None else 0,
                             ptr(c_peer) if not isinstance(c_peer, int) else c_peer, m, n, k,
                             out_dtype == torch.bfloat16, sync or {}, ctas, dev,
                             current_stream(dev) if stream is None else stream, cluster, epilogue == "tma")


def gemm_reference(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Plain PyTorch fp32 reference of the op."""
    return a.float() @ b.float().t()


ACTIVATIONS = ("none", "relu", "gelu", "silu")   # index = the kernel's activation code


def _check_operands(a: torch.Tensor, b: torch.Tensor) -> None:
    if a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16:
        raise TypeError("bf16 operands expected")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[1]:
        raise ValueError("expected A[M,K] and B[N,K]")


def gemm_reduce_scatter(a: torch.Tensor, b: torch.Tensor, shards: Sequence[PtrLike], rank: int, *,
                        done_flags: Sequence[int] = (), done_epoch: int = 0, ticket: int = 0, ticket_base: int = 0,
                        ctas: int = 0, stream: Optional[int] = None, cluster: int = 0, c_multicast: int = 0,
                        out_dtype: torch.dtype = torch.float32, epilogue: str = "red") -> int:
    """K-gemm-rs (csrc/kernels/gemm_collective.cu): ``A[M,K_r] @ B[N,K_r].T`` is this rank's partial sum; the
    epilogue adds every 128x256 tile into ``shards[owner]`` (fp32 ``[M/world, N]``, peer-mapped pointers or local
    tensors, one per rank, zeroed by their owners) with ``red.global.add.v4.f32`` over NVLink.  When
    ``done_flags`` (one word per rank) are given, the last CTA publishes ``done_epoch`` on all of them.
    ``c_multicast`` (the NVLS multicast address of a zeroed fp32 ``[M, N]`` buffer that exists on every rank) turns
    the step into GEMM -> all-reduce: every tile is added into all copies by the switch (``multimem.red``);
    ``shards`` then only tells the world size.  ``out_dtype=torch.bfloat16``: bf16 shards, ``REDG.E.ADD.BF16x8`` —
    half the NVLink bytes, every one of the P additions rounds to bf16.  ``epilogue="tma"`` (fp32 shards): the
    additions are issued by the TMA unit, one ``cp.reduce.async.bulk.tensor.2d`` per 32x32 piece staged in swizzled
    shared memory, instead of ``REDG`` requests from the LSU (``"red"``).
    Subnormal fp32 sums: the ``"red"`` epilogue's ``REDG.E.ADD.F32x4.FTZ.RN`` flushes subnormal values to +-0, so a
    shard element whose partial sums are all below 2^-126 ends as 0 where ``gemm_reference`` keeps it; the ``"tma"``
    epilogue's ``cp.reduce.async.bulk`` keeps them exactly (both measured on an H100, tests/test_gpu_gemm_numerics.py).
    Returns the CTAs launched."""
    if epilogue not in ("red", "tma"):
        raise ValueError("epilogue must be 'red' or 'tma'")
    _check_operands(a, b)
    world = len(shards)
    m, k = a.shape
    n = b.shape[0]
    if m % (128 * world) or n % 256 or k % 64:
        raise ValueError("M, N, K must be multiples of 128*world, 256, 64")
    if out_dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("out_dtype must be float32 or bfloat16")
    for s in shards:
        if not c_multicast and isinstance(s, torch.Tensor) and (s.dtype != out_dtype or
                                                                  tuple(s.shape) != (m // world, n)):
            raise ValueError("every shard must be [M/world, N] of out_dtype")
    dev = a.device.index
    return native().gemm_reduce_scatter(ptr(a), ptr(b), [ptr(s) for s in shards], [int(f) for f in done_flags],
                                        done_epoch, ticket, ticket_base, rank, m, n, k, ctas, dev,
                                        current_stream(dev) if stream is None else stream, cluster, int(c_multicast),
                                        out_dtype == torch.bfloat16, epilogue == "tma")


def gemm_all_to_all(a: torch.Tensor, b: torch.Tensor, recv: Sequence[PtrLike], rank: int, *,
                    out_dtype: torch.dtype = torch.float32, done_flags: Sequence[int] = (), done_epoch: int = 0,
                    ticket: int = 0, ticket_base: int = 0, ctas: int = 0, stream: Optional[int] = None,
                    cluster: int = 0) -> int:
    """K-gemm-a2a: ``C_r = A[M,K] @ B[N,K].T``; row block q of ``C_r`` (``M/world`` rows) is stored by the epilogue
    into slot ``rank`` of ``recv[q]`` (``[world, M/world, N]`` of ``out_dtype``, peer-mapped pointers or local
    tensors).  The all-to-all of expert outputs going home / a Ulysses swap, fused into the producing GEMM."""
    _check_operands(a, b)
    world = len(recv)
    m, k = a.shape
    n = b.shape[0]
    if m % (128 * world) or n % 256 or k % 64:
        raise ValueError("M, N, K must be multiples of 128*world, 256, 64")
    if out_dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("out_dtype must be float32 or bfloat16")
    for r in recv:
        if isinstance(r, torch.Tensor) and (r.dtype != out_dtype or r.numel() != m * n):
            raise ValueError("every receive buffer must be [world, M/world, N] of out_dtype")
    dev = a.device.index
    return native().gemm_all_to_all(ptr(a), ptr(b), [ptr(r) for r in recv], out_dtype == torch.bfloat16,
                                    [int(f) for f in done_flags], done_epoch, ticket, ticket_base, rank, m, n, k, ctas,
                                    dev, current_stream(dev) if stream is None else stream, cluster)


def allgather_gemm(a_full: torch.Tensor, a_src: Sequence[PtrLike], b: torch.Tensor, c: torch.Tensor, rank: int, *,
                   ready: PtrLike = 0, ready_base: int = 0, chunk_bytes: int = 0, done_flags: Sequence[int] = (),
                   done_epoch: int = 0, ticket: int = 0, ticket_base: int = 0, timeout_ns: int = 0, status: int = 0,
                   ctas: int = 0, stream: Optional[int] = None, cluster: int = 0, activation: str = "none") -> int:
    """K-ag-gemm: ``C[M,N] = A[M,K] @ B[N,K].T`` where rank ``q`` holds rows ``[q*M/world, (q+1)*M/world)`` of A.
    ``a_full`` is the local gathered A (this rank's rows already in place), ``a_src[q]`` the peer-mapped address of
    rank q's row block.  One gather thread per CTA pulls the remote rows with TMA bulk copies while the tiles of the
    rows that are already here run on the tensor cores; ``ready`` (int32 ``[M/128]``) counts arrivals per 128-row
    block and counts up forever: pass the value before the launch as ``ready_base`` (it grows by
    ``native().allgather_gemm_chunks_per_block(K, chunk_bytes)`` per launch).  The sources are arbitrary row-block
    pointers, so an all-to-all followed by a GEMM (MoE dispatch -> expert GEMM) is the same call with
    ``a_src[q]`` = slot ``rank`` of rank q's send buffer.  ``activation`` (``none | relu | gelu | silu``; gelu in its
    tanh form) is applied to the fp32 accumulator in the epilogue, before C is rounded and stored.
    Returns the CTAs launched."""
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {ACTIVATIONS}")
    _check_operands(a_full, b)
    world = len(a_src)
    m, k = a_full.shape
    n = b.shape[0]
    if m % (128 * world) or n % 256 or k % 64:
        raise ValueError("M, N, K must be multiples of 128*world, 256, 64")
    if c.dtype not in (torch.float32, torch.bfloat16) or tuple(c.shape) != (m, n):
        raise ValueError("c must be fp32 or bf16 [M, N]")
    if world > 1 and isinstance(ready, torch.Tensor) and (ready.dtype != torch.int32 or ready.numel() < m // 128):
        raise ValueError("ready must be int32 with one word per 128-row block")
    for s in a_src:
        if isinstance(s, torch.Tensor) and (s.dtype != torch.bfloat16 or s.numel() != m // world * k):
            raise ValueError("every a_src row block must be bf16 with M/world * K elements")
    dev = a_full.device.index
    return native().allgather_gemm(ptr(a_full), [ptr(s) for s in a_src], ptr(b), ptr(c), c.dtype == torch.bfloat16,
                                   ptr(ready), ready_base, chunk_bytes, [int(f) for f in done_flags], done_epoch,
                                   ticket, ticket_base, timeout_ns, status, rank, m, n, k, ctas, dev,
                                   current_stream(dev) if stream is None else stream, cluster,
                                   ACTIVATIONS.index(activation))
