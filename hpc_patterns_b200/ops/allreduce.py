"""Allreduce building blocks (csrc/kernels/ring_allreduce.cu) on tensors or raw addresses.

``accumulate`` is the reference's ``Accumulate`` kernel (allreduce-mpi-sycl.cpp:26-31);
``ring_allreduce`` / ``two_shot`` / ``nvls`` are the fused one-launch replacements of its
``SendRecvRing`` loop and ``MPI_Allreduce``.  The multi-rank drivers live in
``hpc_patterns_b200.models.allreduce``; these wrappers are what they (and the tests) call.

The value-index pair types of maxloc / minloc (``float_int``, ``double_int``, ``long_int``, ``2int``, ``short_int``, ↔
MPI_FLOAT_INT ...) are C structs ``{value; int index;}`` in their natural layout; ``pack_loc`` / ``unpack_loc`` convert
between that layout (a flat uint8 tensor, padding zero) and a (values, int32 indices) pair of tensors.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import native
from ._util import current_stream, ptr

_DTYPE_NAME = {torch.float32: "float", torch.int32: "int", torch.bfloat16: "bfloat16", torch.float16: "half"}


def dtype_name(t: torch.Tensor) -> str:
    try:
        return _DTYPE_NAME[t.dtype]
    except KeyError:
        raise TypeError(f"allreduce kernels support float32, int32, bfloat16 and float16, not {t.dtype}") from None


# pair type -> (torch dtype of the value, bytes per pair, byte offset of the index)
LOC_LAYOUT = {"float_int": (torch.float32, 8, 4), "double_int": (torch.float64, 16, 8), "long_int": (torch.int64, 16, 8),
              "2int": (torch.int32, 8, 4), "short_int": (torch.int16, 8, 4)}
_LOC_OF_VALUE = {vt: name for name, (vt, _, _) in LOC_LAYOUT.items()}


def pack_loc(values: torch.Tensor, indices: torch.Tensor, dtype: Optional[str] = None) -> torch.Tensor:
    """The pairs (values[i], indices[i]) in the C layout of ``dtype`` (by default the pair type of ``values.dtype``):
    a flat uint8 tensor on ``values``' device, padding bytes zero.  Indices are converted to int32."""
    if dtype is None:
        if values.dtype not in _LOC_OF_VALUE:
            raise TypeError(f"no value-index pair type has {values.dtype} values")
        dtype = _LOC_OF_VALUE[values.dtype]
    if dtype not in LOC_LAYOUT:
        raise ValueError(f"dtype must be one of {tuple(LOC_LAYOUT)}, not {dtype!r}")
    vt, size, off = LOC_LAYOUT[dtype]
    if values.numel() != indices.numel():
        raise ValueError("values and indices must have the same number of elements")
    n = values.numel()
    buf = torch.zeros(n, size, dtype=torch.uint8, device=values.device)
    vbytes = values.reshape(-1).to(vt).contiguous().view(torch.uint8).reshape(n, -1)
    buf[:, :vbytes.shape[1]] = vbytes
    buf[:, off:off + 4] = indices.reshape(-1).to(torch.int32).to(values.device).contiguous().view(torch.uint8) \
        .reshape(n, 4)
    return buf.reshape(-1)


def unpack_loc(buf: torch.Tensor, dtype: str):
    """(values, int32 indices) of the pairs of type ``dtype`` held in ``buf`` (any tensor whose bytes are the pairs)."""
    if dtype not in LOC_LAYOUT:
        raise ValueError(f"dtype must be one of {tuple(LOC_LAYOUT)}, not {dtype!r}")
    vt, size, off = LOC_LAYOUT[dtype]
    b = buf.contiguous().reshape(-1).view(torch.uint8).reshape(-1, size)
    vbytes = torch.empty(0, dtype=vt).element_size()
    return (b[:, :vbytes].contiguous().view(vt).reshape(-1), b[:, off:off + 4].contiguous().view(torch.int32).reshape(-1))


def loc_combine(a: torch.Tensor, b: torch.Tensor, dtype: str, op: str) -> torch.Tensor:
    """a o b for the packed pairs ``a`` and ``b`` (pack_loc) with the kernels' rules: the larger (maxloc) or smaller
    (minloc) value wins, a NaN value wins in both and -0 < +0; bit-equal values or two NaNs take the smaller index; the
    result is packed with zero padding and the canonical NaN (all bits set but the sign)."""
    va, ia = unpack_loc(a, dtype)
    vb, ib = unpack_loc(b, dtype)
    mx = op == "maxloc"
    if va.is_floating_point():
        na, nb = torch.isnan(va), torch.isnan(vb)
        sa, sb = torch.signbit(va), torch.signbit(vb)
        eq = (va == vb) & (sa == sb)
        gt = (va > vb) | ((va == vb) & sb & ~sa)       # in the order -0 < +0
        better = (na & ~nb) | (~na & ~nb & ~eq & (gt if mx else ~gt))
        tie = (na & nb) | (~na & ~nb & eq)
    else:
        better = va > vb if mx else va < vb
        tie = va == vb
    take_a = better | (tie & (ia <= ib))
    v = torch.where(take_a, va, vb)
    if v.is_floating_point():
        bits = torch.int32 if v.dtype == torch.float32 else torch.int64
        canon = torch.tensor(0x7FFFFFFF if bits == torch.int32 else 0x7FFFFFFFFFFFFFFF, dtype=bits).view(v.dtype)
        v = torch.where(torch.isnan(v), canon.to(v.device), v)
    return pack_loc(v, torch.where(take_a, ia, ib), dtype)


def accumulate(va: torch.Tensor, vc: torch.Tensor, stream: Optional[int] = None) -> torch.Tensor:
    """vc += va (in place) with the native kernel; returns vc."""
    if va.shape != vc.shape or va.dtype != vc.dtype:
        raise ValueError("va and vc must have the same shape and dtype")
    dev = vc.device.index
    native().accumulate(ptr(va), ptr(vc), vc.numel(), dtype_name(vc),
                        current_stream(dev) if stream is None else stream)
    return vc


def accumulate_reference(va: torch.Tensor, vc: torch.Tensor) -> torch.Tensor:
    """Plain PyTorch reference of the same op."""
    return vc + va


def init3(va: Optional[torch.Tensor], vb: Optional[torch.Tensor], vc: Optional[torch.Tensor],
          a: float, b: float, c: float, stream: Optional[int] = None) -> None:
    ref = next(t for t in (va, vb, vc) if t is not None)
    dev = ref.device.index
    native().init3(ptr(va) if va is not None else 0, ptr(vb) if vb is not None else 0,
                   ptr(vc) if vc is not None else 0, ref.numel(), a, b, c, dtype_name(ref),
                   current_stream(dev) if stream is None else stream)


def count_mismatch(v: torch.Tensor, expected: float, stream: Optional[int] = None) -> int:
    dev = v.device.index
    count = torch.zeros(1, dtype=torch.int64, device=v.device)
    native().count_mismatch(ptr(v), v.numel(), float(expected), dtype_name(v), count.data_ptr(),
                            current_stream(dev) if stream is None else stream)
    torch.cuda.synchronize(dev)
    return int(count.item())


# -------------------------------------------------------------------------------------------------- reduce-scatter ----
# ``reduce_scatter`` is the one-launch reduce-scatter (↔ MPI_Reduce_scatter_block, ncclReduceScatter,
# reduce_scatter_tensor): rank p's send buffer holds P segments of n elements; afterwards rank r's receive buffer (n
# elements) holds op over p of segment r of rank p's send buffer, owner first in every element,
# ((S_r[r] o S_{r+1}[r]) o ...) o S_{r+P-1}[r].  Any op the allreduce takes for the type, with its refusals.
# The refusal words and the element sizes are the native module's (csrc/kernels/api.h), read from it.
RS_MAX_RANKS = 16


def check_reduce_scatter_args(world: int, n: int, dtype: str) -> None:
    """ValueError with the native words if the launcher would refuse (world, n, dtype).  An op that does not reduce the
    type is refused by the launcher with dispatch_op's words (``models.allreduce.check_op_type`` says them first)."""
    C = native()
    if n <= 0 or n * C.elem_size(dtype) % 16:     # elem_size: ValueError for a name that is not a type
        raise ValueError(C.REDUCE_SCATTER_COUNT_ERROR)
    if not 1 <= world <= RS_MAX_RANKS:
        raise ValueError(C.REDUCE_SCATTER_WORLD_ERROR)


def reduce_scatter(send, recv: int, pads, ticket: int, ticket_base: int, rank: int, n: int, barrier_epoch: int,
                   timeout_ns: int = 0, status: int = 0, dtype: str = "float", ctas: int = 0, device: int = 0,
                   stream: int = 0, op: str = "sum") -> int:
    """Enqueue one reduce-scatter of rank ``rank`` on ``stream``.  ``send`` / ``pads`` are every rank's peer-mapped
    addresses, ``recv`` this rank's receive buffer of ``n`` elements.  Returns the CTAs launched (advance the ticket
    counter by it)."""
    world = len(send)
    check_reduce_scatter_args(world, n, dtype)
    if len(pads) != world:
        raise ValueError("reduce-scatter: inconsistent rank lists")
    if not 0 <= rank < world:
        raise ValueError("reduce-scatter: rank out of range")
    seg = n * native().elem_size(dtype)
    if not (send[rank] + world * seg <= recv or recv + seg <= send[rank]):
        raise ValueError(native().REDUCE_SCATTER_OVERLAP_ERROR)
    return native().reduce_scatter(list(send), recv, list(pads), ticket, ticket_base & 0xFFFFFFFF, rank, n,
                                   barrier_epoch, timeout_ns, status, dtype, ctas, device, stream, op)


def reduce_scatter_reference(sends, op: str, dtype: str):
    """Rank r's receive buffer for every r, computed in torch / Python from the send buffers (each P segments of n
    elements; pair types: packed bytes), owner first: ((S_r[r] o S_{r+1}[r]) o ...).  The 16-bit floating sum and prod
    accumulate in fp32 and round once.  torch's min / max may keep the other zero of a +0 / -0 tie and its NaNs are not
    the kernels' canonical ones; everything else is the kernels' result bit for bit (integers wrap)."""
    world = len(sends)
    if dtype in LOC_LAYOUT:
        parts = [s.contiguous().view(torch.uint8).reshape(world, -1) for s in sends]
        out = []
        for r in range(world):
            acc = parts[r][r].clone()
            for k in range(1, world):
                acc = loc_combine(acc, parts[(r + k) % world][r], dtype, op)
            out.append(acc)
        return out
    parts = [s.reshape(world, -1) for s in sends]
    lowp = parts[0].dtype in (torch.bfloat16, torch.float16) and op in ("sum", "prod")
    out = []
    for r in range(world):
        acc = parts[r][r].float() if lowp else parts[r][r].clone()
        for k in range(1, world):
            x = parts[(r + k) % world][r]
            acc = _combine_ref(acc, x.float() if lowp else x, op)
        out.append(acc.to(parts[0].dtype) if lowp else acc)
    return out


def _combine_ref(a: torch.Tensor, b: torch.Tensor, op: str) -> torch.Tensor:
    if op == "sum":
        return a + b
    if op in ("prod", "product"):
        return a * b
    if op in ("min", "max"):
        return torch.minimum(a, b) if op == "min" else torch.maximum(a, b)
    if op in ("band", "bor", "bxor"):
        return {"band": torch.bitwise_and, "bor": torch.bitwise_or, "bxor": torch.bitwise_xor}[op](a, b)
    if op in ("land", "lor", "lxor"):
        f = {"land": torch.logical_and, "lor": torch.logical_or, "lxor": torch.logical_xor}[op]
        return f(a != 0, b != 0).to(a.dtype)
    raise ValueError(f"unknown op {op!r}")
