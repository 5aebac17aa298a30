"""Element-wise oracle of the bitwise and logical allreduce ops (band, bor, bxor, land, lor, lxor;
csrc/kernels/ring_allreduce_ops.cu): data, expected results and the constant-data check of the miniapps.

All six ops are exact, commutative and associative, so every algorithm (the rings, ring-rsag, two-shot, the unfused
ring's combine) and every rank computes the same bits: one fold of VA over the ranks, and VA itself at one rank.

* ``band`` / ``bor`` / ``bxor``: ``&``, ``|``, ``^`` of the element bits, whatever the width and signedness;
* ``land`` / ``lor`` / ``lxor``: an element is true iff it is nonzero over its WHOLE width (a long holding 1 << 40 is
  true), and a result over two or more ranks is 0 or 1 of the type.

Integers only: the floating types are refused by every layer.  Bits are numpy unsigned arrays, tensors the dtypes of
tests/reduce_op_oracle.py (unsigned integers stored in the signed torch type of their width).
"""
from __future__ import annotations

from typing import List

import numpy as np
import torch

from tests.reduce_op_oracle import _UBITS, TORCH_DTYPE, elem_bytes, from_bits, to_bits
from tests.rsag_oracle import segment

INT_TYPES = ("int", "uint", "long", "ulong", "short", "ushort", "uchar")
FLOAT_TYPES = ("float", "double", "bfloat16", "half")
BIT_OPS = ("band", "bor", "bxor", "land", "lor", "lxor")
LOGICAL_OPS = ("land", "lor", "lxor")
KINDS = ("dense", "sparse", "high")


def combine(a: np.ndarray, b: np.ndarray, op: str, dtype: str) -> np.ndarray:
    """op(a, b) lane by lane on raw bits."""
    ub = _UBITS[elem_bytes(dtype)]
    a = a.astype(ub, copy=False)
    b = b.astype(ub, copy=False)
    if op == "band":
        return a & b
    if op == "bor":
        return a | b
    if op == "bxor":
        return a ^ b
    if op == "land":
        return ((a != 0) & (b != 0)).astype(ub)
    if op == "lor":
        return ((a != 0) | (b != 0)).astype(ub)
    if op == "lxor":
        return ((a != 0) ^ (b != 0)).astype(ub)
    raise ValueError(f"unknown op {op!r}")


def fold(parts: List[np.ndarray], op: str, dtype: str) -> np.ndarray:
    """parts[0] o parts[1] o ...; parts[0] itself, unnormalised, for one part."""
    acc = parts[0].astype(_UBITS[elem_bytes(dtype)], copy=True)
    for p in parts[1:]:
        acc = combine(acc, p, op, dtype)
    return acc


def allreduce_expected(vas: List[torch.Tensor], op: str, dtype: str) -> torch.Tensor:
    """VC of every rank after any allreduce algorithm."""
    return from_bits(fold([to_bits(v) for v in vas], op, dtype), dtype)


def reduce_scatter_expected(vas: List[torch.Tensor], s: int, op: str, dtype: str) -> torch.Tensor:
    """Segment ``s`` of the reduce-scatter phase of ring-rsag."""
    return allreduce_expected(vas, op, dtype)[segment(vas[0].numel(), len(vas), s)]


def combine_expected(vc: torch.Tensor, va: torch.Tensor, op: str, dtype: str) -> torch.Tensor:
    """VC after the combine kernel: op(VC, VA)."""
    return from_bits(combine(to_bits(vc), to_bits(va), op, dtype), dtype)


def brute_force(values: List[List[int]], op: str, dtype: str) -> List[int]:
    """The same fold on Python ints, one element at a time: ``values[r][i]`` is element i of rank r, as an unsigned
    integer of the type's width."""
    mask = (1 << 8 * elem_bytes(dtype)) - 1
    out = []
    for column in zip(*values):
        acc = column[0]
        for x in column[1:]:
            if op == "band":
                acc &= x
            elif op == "bor":
                acc |= x
            elif op == "bxor":
                acc ^= x
            elif op == "land":
                acc = int(acc != 0 and x != 0)
            elif op == "lor":
                acc = int(acc != 0 or x != 0)
            elif op == "lxor":
                acc = int((acc != 0) != (x != 0))
            else:
                raise ValueError(f"unknown op {op!r}")
        out.append(acc & mask)
    return out


# ------------------------------------------------------------------- inputs ----
def make_inputs(world: int, n: int, dtype: str, seed: int, kind: str) -> List[torch.Tensor]:
    """VA of every rank (``n`` elements each), different per rank, per element and per ``seed``.

    ``dense``   random bits over the whole width;
    ``sparse``  zero-heavy: per element every rank zero, every rank nonzero, exactly one rank nonzero, or each rank
                nonzero at random, so that every logical result takes both 0 and 1 at every rank count; the nonzero
                values are random bits, single bits among them;
    ``high``    as ``sparse``, with nonzero values that are nonzero only in their top byte or, in 64-bit lanes, only in
                their top 32 bits: a logical op that tests truth per byte or per 32-bit word instead of per element
                gets them, or the zeros next to them, wrong."""
    if dtype not in INT_TYPES:
        raise ValueError(f"the bitwise and logical ops reduce integer types only, not {dtype}")
    rng = np.random.default_rng(0xB170000 + seed)
    nb = elem_bytes(dtype)
    ub = _UBITS[nb]
    bits = 8 * nb

    def random_bits(size):
        raw = rng.integers(0, 1 << 62, size, dtype=np.uint64) * 4 + rng.integers(0, 4, size, dtype=np.uint64)
        return raw.astype(ub)

    def nonzero(size):
        if kind == "sparse":
            v = random_bits(size)
            single = rng.integers(0, 4, size) == 0
            v[single] = (np.uint64(1) << rng.integers(0, bits, int(single.sum())).astype(np.uint64)).astype(ub)
        else:                                               # high part only
            top = rng.integers(1, 256, size, dtype=np.uint64) << np.uint64(bits - 8)
            if nb == 8:
                hi32 = (rng.integers(1, 1 << 32, size, dtype=np.uint64) << np.uint64(32))
                top = np.where(rng.integers(0, 2, size) == 0, top, hi32)
            v = top.astype(ub)
        v[v == 0] = ub(1 << (bits - 1))
        return v

    if kind == "dense":
        return [from_bits(random_bits(n), dtype) for _ in range(world)]
    if kind not in ("sparse", "high"):
        raise ValueError(f"unknown kind {kind!r}")
    mode = rng.integers(0, 4, n)                            # 0 all zero, 1 all nonzero, 2 one nonzero, 3 random
    one = rng.integers(0, world, n)
    out = []
    for r in range(world):
        live = (mode == 1) | ((mode == 2) & (one == r)) | ((mode == 3) & (rng.integers(0, 2, n) == 0))
        out.append(from_bits(np.where(live, nonzero(n), ub(0)), dtype))
    return out


# ------------------------------------------------------ constant-data check ----
# What the miniapps (bin/allreduce, AllreduceMiniapp.run) give every rank and expect back, exact in uchar up to 16
# ranks; each bitwise op's result differs from its logical twin's from 2 ranks on, and VC before the run differs from
# the result, so a VC that is never written shows.
def check_input(op: str, rank: int) -> int:
    return {"band": 255 - (1 << rank % 4), "bor": 1 << rank % 4, "bxor": 128 if rank == 0 else rank,
            "land": rank + 1, "lor": 2 * (rank % 2), "lxor": 3 if rank == 0 else 0}[op]


def check_expected(op: str, world: int) -> int:
    if op == "band":
        return 256 - (1 << min(world, 4))
    if op == "bor":
        return (1 << min(world, 4)) - 1
    if op == "bxor":
        x = 128
        for r in range(1, world):
            x ^= r
        return x
    if op == "land":
        return 1
    if op == "lor":
        return 1 if world >= 2 else 0
    return 1 if world >= 2 else 3                           # lxor: one rank gives VA itself


CHECK_VC = {"band": 0, "bor": 16, "bxor": 64, "land": 0, "lor": 3, "lxor": 5}


def mismatches(got: torch.Tensor, want: torch.Tensor) -> int:
    """Elements whose bits differ."""
    if got.shape != want.shape or got.dtype != want.dtype:
        raise ValueError(f"shape/dtype differ: {tuple(got.shape)} {got.dtype} vs {tuple(want.shape)} {want.dtype}")
    return int((to_bits(got) != to_bits(want)).sum())
