"""Element-wise oracle of the prod / min / max allreduce kernels (csrc/kernels/ring_allreduce_ops.cu): data, expected
results and the bit comparison the GPU tests assert on.  numpy for the arithmetic, torch tensors in and out.

What each algorithm computes (docs/allreduce.md), with ``o`` the op:

* the fused ring (push and pull, both slot policies) and the unfused ring: ``ring_expected`` -- rank r holds
  ((VA[r] o VA[r-1]) o VA[r-2]) o ..., VC overwritten (never read);
* ring-rsag: ``rsag_expected`` / ``reduce_scatter_expected`` -- segment s is ((VA[s+1] o VA[s+2]) o ...) o VA[s];
* two-shot: ``two_shot_expected`` -- slice s is ((VA[s] o VA[s+1]) o ...) (ranks mod P, owner first) in every element;
  the 16-bit prod multiplies in fp32 and rounds once;
* combine (the unfused ring's kernel): ``combine(vc, va, op, dtype)``.

Semantics: integers compare with their own signedness and multiply modulo 2^w; floats follow IEEE 754-2019 maximum /
minimum (a NaN input gives NaN; -0 < +0) and round every product to nearest even without flushing subnormals; the
16-bit floats do the same in their own format.  Every NaN result is the canonical quiet NaN: all bits set but the
sign (0x7fff, 0x7fffffff, 0x7fffffffffffffff), so ``mismatches`` compares raw bits with no NaN exception.
"""
from __future__ import annotations

from typing import List

import numpy as np
import torch

from tests.lowp_allreduce_oracle import round16
from tests.rsag_oracle import segment

TYPES = ("float", "int", "uint", "double", "long", "ulong", "short", "ushort", "uchar", "bfloat16", "half")
OPS = ("prod", "min", "max")
FLOATS = ("float", "double", "bfloat16", "half")
# element type -> the torch dtype the tests store it as (unsigned integers in the signed type of their width: the
# kernels only see bits) and the numpy dtype its values are computed in (bfloat16: fp32 values of its bits)
TORCH_DTYPE = {"float": torch.float32, "int": torch.int32, "uint": torch.int32, "double": torch.float64,
               "long": torch.int64, "ulong": torch.int64, "short": torch.int16, "ushort": torch.int16,
               "uchar": torch.uint8, "bfloat16": torch.bfloat16, "half": torch.float16}
_NP = {"float": np.float32, "int": np.int32, "uint": np.uint32, "double": np.float64, "long": np.int64,
       "ulong": np.uint64, "short": np.int16, "ushort": np.uint16, "uchar": np.uint8, "half": np.float16}
_UBITS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
_SBITS = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}
_TBITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def elem_bytes(dtype: str) -> int:
    return torch.empty((), dtype=TORCH_DTYPE[dtype]).element_size()


def lanes(dtype: str) -> int:
    return 16 // elem_bytes(dtype)


def canonical_nan(dtype: str) -> int:
    return (1 << (8 * elem_bytes(dtype) - 1)) - 1


# ------------------------------------------------------------ representations ----
def to_bits(t: torch.Tensor) -> np.ndarray:
    """Raw bits of a tensor as an unsigned numpy array."""
    return t.contiguous().view(_TBITS[t.element_size()]).numpy().view(_UBITS[t.element_size()]).copy()


def from_bits(b: np.ndarray, dtype: str) -> torch.Tensor:
    """A tensor of ``dtype`` (its TORCH_DTYPE) holding the bits ``b``."""
    nb = elem_bytes(dtype)
    ub = np.ascontiguousarray(b.astype(_UBITS[nb], copy=False))
    return torch.from_numpy(ub.view(_SBITS[nb]).copy()).view(TORCH_DTYPE[dtype])


def values(b: np.ndarray, dtype: str) -> np.ndarray:
    """The numeric values of bits ``b`` (bfloat16 as exact fp32)."""
    if dtype == "bfloat16":
        return (b.astype(np.uint32) << 16).view(np.float32)
    return b.view(_NP[dtype])


def _bits_of(v: np.ndarray, dtype: str) -> np.ndarray:
    return np.ascontiguousarray(v.astype(_NP[dtype], copy=False)).view(_UBITS[elem_bytes(dtype)])


def _round16_bits(x: np.ndarray, dtype: str) -> np.ndarray:
    """fp64 values rounded once to the 16-bit type, as bits (NaN canonical)."""
    b = to_bits(round16(x, dtype))
    return np.where(np.isnan(x), np.uint16(canonical_nan(dtype)), b)


# ------------------------------------------------------------------ combine ----
def combine(a: np.ndarray, b: np.ndarray, op: str, dtype: str) -> np.ndarray:
    """op(a, b) lane by lane on raw bits (``a`` is the accumulated side), with the kernels' semantics."""
    a = a.astype(_UBITS[elem_bytes(dtype)], copy=False)
    b = b.astype(_UBITS[elem_bytes(dtype)], copy=False)
    x, y = values(a, dtype), values(b, dtype)
    nan_bits = a.dtype.type(canonical_nan(dtype))
    if op == "prod":
        if dtype not in FLOATS:
            return a * b                                        # unsigned: wraps modulo 2^w, no warning
        with np.errstate(all="ignore"):
            if dtype in ("bfloat16", "half"):                   # the fp64 product of two 16-bit values is exact
                return _round16_bits(x.astype(np.float64) * y.astype(np.float64), dtype)
            r = _bits_of(x * y, dtype)                          # IEEE binary32 / binary64, round to nearest even
        return np.where(np.isnan(x) | np.isnan(y) | np.isnan(values(r, dtype)), nan_bits, r)
    if op not in ("min", "max"):
        raise ValueError(f"unknown op {op!r}")
    big = op == "max"
    with np.errstate(invalid="ignore"):
        pick_a = x > y if big else x < y
    r = np.where(pick_a, a, b)
    if dtype in FLOATS:
        eq = x == y                                             # +0 == -0: AND keeps +0 (max), OR keeps -0 (min)
        r = np.where(eq, a & b if big else a | b, r)
        r = np.where(np.isnan(x) | np.isnan(y), nan_bits, r)
    return r


def _prod16_f32(parts: List[np.ndarray], dtype: str) -> np.ndarray:
    """Two-shot's 16-bit prod: fp32 products in the given order, rounded once to the 16-bit type."""
    acc = values(parts[0], dtype).astype(np.float32)
    with np.errstate(all="ignore"):
        for p in parts[1:]:
            acc = acc * values(p, dtype).astype(np.float32)
    return _round16_bits(acc.astype(np.float64), dtype)


# ----------------------------------------------------------------- orders ----
def _fold(parts: List[np.ndarray], op: str, dtype: str) -> np.ndarray:
    acc = parts[0]
    for p in parts[1:]:
        acc = combine(acc, p, op, dtype)
    return acc


def ring_expected(vas: List[torch.Tensor], rank: int, op: str, dtype: str) -> torch.Tensor:
    """VC of ``rank`` after the fused or unfused ring: ((VA[rank] o VA[rank-1]) o ...) o VA[rank-P+1]."""
    world = len(vas)
    return from_bits(_fold([to_bits(vas[(rank - t) % world]) for t in range(world)], op, dtype), dtype)


def reduce_scatter_expected(vas: List[torch.Tensor], s: int, op: str, dtype: str) -> torch.Tensor:
    """Segment ``s`` as rank ``s`` reduces it: ((VA[s+1] o VA[s+2]) o ...) o VA[s]."""
    world = len(vas)
    seg = segment(vas[0].numel(), world, s)
    return from_bits(_fold([to_bits(vas[(s + k) % world][seg]) for k in range(1, world + 1)], op, dtype), dtype)


def rsag_expected(vas: List[torch.Tensor], op: str, dtype: str) -> torch.Tensor:
    """VC of every rank after the reduce-scatter + all-gather ring."""
    return torch.cat([reduce_scatter_expected(vas, s, op, dtype) for s in range(len(vas))])


def two_shot_expected(vas: List[torch.Tensor], op: str, dtype: str) -> torch.Tensor:
    """VC of every rank after two-shot: slice s is ((VA[s] o VA[s+1]) o ...), owner first in every element."""
    world = len(vas)
    out = []
    for s in range(world):
        seg = segment(vas[0].numel(), world, s)
        parts = [to_bits(vas[(s + q) % world][seg]) for q in range(world)]
        out.append(_prod16_f32(parts, dtype) if op == "prod" and dtype in ("bfloat16", "half")
                   else _fold(parts, op, dtype))
    return from_bits(np.concatenate(out), dtype)


def combine_expected(vc: torch.Tensor, va: torch.Tensor, op: str, dtype: str) -> torch.Tensor:
    """VC after the combine kernel: op(VC, VA)."""
    return from_bits(combine(to_bits(vc), to_bits(va), op, dtype), dtype)


# ------------------------------------------------------------------- inputs ----
def kinds(op: str, dtype: str) -> tuple:
    """The input kinds that apply to (op, dtype)."""
    if op == "prod":
        return ("wrap",) if dtype not in FLOATS else ("near-one", "subnormal", "overflow")
    return ("full", "special") if dtype in FLOATS else ("full", "extremes")


def make_inputs(world: int, n: int, dtype: str, seed: int, op: str, kind: str) -> List[torch.Tensor]:
    """VA of every rank (``n`` elements each), different per rank, per element and per ``seed``.

    min / max:
      ``full``      random bits over the whole range (floats: random finite values of every magnitude and sign), with
                    many duplicates across ranks (ties between equal values, and between +0 and -0, must resolve);
      ``special``   (floats) +-0, +-inf, NaN and ordinary values mixed in every lane;
      ``extremes``  (integers) 0, 1, all-ones, the top bit alone (0x80..0) and its neighbours: a signed / unsigned
                    confusion reverses their order.
    prod:
      ``near-one``  floats in [0.5, 2) with random signs and mantissas, so P products round but stay finite;
      ``subnormal`` floats whose products land in the subnormal range (an FTZ multiply flushes them to zero);
      ``overflow``  floats large enough that products overflow to +-inf, with some zeros (inf * 0 = NaN);
      ``wrap``      (integers) random bits: products wrap modulo 2^w."""
    rng = np.random.default_rng(0x0B5E0000 + seed)
    nb = elem_bytes(dtype)
    ub = _UBITS[nb]
    out = []
    pool = rng.integers(0, 1 << 62, max(8, n // 4), dtype=np.uint64)   # shared values: duplicates across ranks
    for r in range(world):
        if kind in ("full", "wrap"):
            raw = rng.integers(0, 1 << 62, n, dtype=np.uint64) * 4 + rng.integers(0, 4, n, dtype=np.uint64)
            dup = rng.integers(0, 3, n) == 0
            raw[dup] = pool[rng.integers(0, pool.size, int(dup.sum()))]
            b = raw.astype(ub)                                  # truncate: random bits of the width
            if dtype in FLOATS:                                 # finite values only: NaN / inf go in "special"
                v = values(b, dtype)
                b = np.where(np.isfinite(v), b, b & ub(~(1 << (8 * nb - 2)) & ((1 << 8 * nb) - 1)))
        elif kind == "extremes":
            top = 1 << (8 * nb - 1)
            cands = np.array([0, 1, 2, top - 1, top, top + 1, (1 << 8 * nb) - 1, (1 << 8 * nb) - 2], dtype=np.uint64)
            b = cands[rng.integers(0, cands.size, n)].astype(ub)
        elif kind == "special":
            vals = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 1.5, -2.5], dtype=np.float64)
            v = vals[rng.integers(0, vals.size, n)]
            b = _round16_bits(v, dtype) if dtype in ("bfloat16", "half") else _bits_of(v, dtype)
            nan = np.isnan(v) & (rng.integers(0, 2, n) == 0)   # some NaNs negative or with a payload
            b = np.where(nan, b | ub(1 << (8 * nb - 1)), b)
        elif kind in ("near-one", "subnormal", "overflow"):
            sign = np.where(rng.integers(0, 2, n) == 0, 1.0, -1.0)
            if kind == "near-one":
                mag = np.ldexp(1.0 + rng.random(n), rng.integers(-1, 1, n))
            elif kind == "subnormal":
                lo = {"float": -126, "double": -1022, "bfloat16": -126, "half": -14}[dtype]
                # two factors near 2^(lo/2): their product lands near 2^lo, at the subnormal boundary
                mag = np.ldexp(1.0 + rng.random(n), lo // 2 + rng.integers(-4, 2, n))
            else:
                hi = {"float": 127, "double": 1023, "bfloat16": 127, "half": 15}[dtype]
                mag = np.ldexp(1.0 + rng.random(n), hi // 2 + rng.integers(-1, 3, n))
                mag[rng.integers(0, 32, n) == 0] = 0.0
            v = sign * mag
            b = _round16_bits(v, dtype) if dtype in ("bfloat16", "half") else _bits_of(v, dtype)
        else:
            raise ValueError(f"unknown kind {kind!r}")
        out.append(from_bits(b, dtype))
    return out


# -------------------------------------------------------------- comparison ----
def mismatches(got: torch.Tensor, want: torch.Tensor) -> int:
    """Elements whose bits differ (NaN compared by its bits: results are canonical)."""
    if got.shape != want.shape or got.dtype != want.dtype:
        raise ValueError(f"shape/dtype differ: {tuple(got.shape)} {got.dtype} vs {tuple(want.shape)} {want.dtype}")
    return int((to_bits(got) != to_bits(want)).sum())


def describe(got: torch.Tensor, want: torch.Tensor, lanes_per_vec: int = 1) -> str:
    """The first differing elements, for assertion messages."""
    g, w = to_bits(got), to_bits(want)
    bad = np.flatnonzero(g != w)[:4].tolist()
    return ", ".join(f"[{i} (vector {i // lanes_per_vec})] got {got[i].item()!r} (0x{int(g[i]):x}) "
                     f"want {want[i].item()!r} (0x{int(w[i]):x})" for i in bad)
