"""Element-wise oracle of the allreduce kernels (csrc/kernels/ring_allreduce.cu) for the 16-bit floating types, bfloat16
and half: data, expected results and the comparison the GPU tests assert on.  Torch and numpy only.

What each algorithm computes (docs/allreduce.md):

* the fused ring (push and pull, both slot policies) and the unfused ring: ``ring_expected`` -- rank r adds VA[r],
  VA[r-1], ... into a zeroed VC, every add rounded to nearest even in the 16-bit type;
* ring-rsag: ``rsag_expected`` / ``reduce_scatter_expected`` / ``all_gather_expected`` -- segment s is
  ((VA[s+1] + VA[s+2]) + ...) + VA[s], one rounded add per hop, the same bits on every rank;
* two-shot: ``two_shot_expected`` -- slice s is the fp32 sum VA[s] + VA[s+1] + ... (ranks mod P, owner first), rounded
  once to the 16-bit type.

The ring expectations are the existing oracles' (tests/allreduce_oracle.py, tests/rsag_oracle.py) applied to bfloat16 /
float16 tensors.  They rest on one fact: torch's CPU ``a + b`` on such tensors is the correctly rounded 16-bit add (it
adds in fp32 and rounds once, and fp32 has more than 2p+2 bits).  ``round16`` is an independent exact rounding of fp64
values, and tests/test_lowp_allreduce_oracle.py checks the fact against it.

The data (``make_inputs``) has every mantissa bit random, random signs and one exponent band per rank, so that sums
really round; ``kind="subnormal"`` lands results in the subnormal range and ``kind="overflow"`` (half) reaches +-inf and
NaN.  ``mismatches`` compares bits, except that any NaN equals any NaN: the GPU's canonical NaN and the CPU's differ.
"""
from __future__ import annotations

from typing import List

import numpy as np
import torch

from tests.allreduce_oracle import bits, ring_expected  # noqa: F401  (re-exported: the ring expectation)
from tests.rsag_oracle import all_gather_expected, reduce_scatter_expected, rsag_expected, segment  # noqa: F401

LOWP = ("bfloat16", "half")
TORCH_DTYPE = {"bfloat16": torch.bfloat16, "half": torch.float16}
LANES = 8                                   # elements per 16-byte vector
# (exponent bits, stored mantissa bits, exponent bias)
FORMAT = {"bfloat16": (8, 7, 127), "half": (5, 10, 15)}
# "full" data: rank r's values lie in the binades 2^(lo + (r * step) % span) ... 2^(lo + (r * step) % span + jitter - 1),
# (lo, step, span, jitter).  The ranks' bands spread over more binades than fp32 has bits beyond the 16-bit mantissa, so
# even fp32 sums round and their order shows; sums of up to 8 values stay far from overflow (|x| < 2^12 bf16, 2^6 fp16).
_FULL_BANDS = {"bfloat16": (-10, 4, 16, 8), "half": (-12, 4, 14, 4)}
# ... and in 1/8 of the elements two random ranks hold +X and -X, X in [2^e, 2^(e+1)): the pair cancels exactly, but every
# small term added while X is in the sum loses its low bits, so the summation ORDER shows even through fp32 (two-shot)
_CANCEL_E = {"bfloat16": 40, "half": 14}


def _from_fields(sign: np.ndarray, exp_field: np.ndarray, mant: np.ndarray, dtype: str) -> torch.Tensor:
    e_bits, m_bits, _ = FORMAT[dtype]
    raw = (sign.astype(np.uint16) << 15) | (exp_field.astype(np.uint16) << m_bits) | mant.astype(np.uint16)
    return torch.from_numpy(raw.view(np.int16).copy()).view(TORCH_DTYPE[dtype])


def make_inputs(world: int, n: int, dtype: str, seed: int, kind: str = "full", device: str = "cpu") -> List[torch.Tensor]:
    """VA of every rank (``n`` elements each), different per rank, per element and per ``seed``.

    ``full``       full-mantissa values with random signs, rank r in its own band of binades (so sums round), and in 1/8
                   of the elements a +X / -X pair on two ranks (so the order of the adds shows, in fp32 too);
    ``subnormal``  exponent field 0 or 1 (the subnormals and the lowest binade) with random signs: many sums and partial
                   sums are subnormal;
    ``overflow``   (half) values in the top binade with random signs: same-sign sums overflow to +-inf, and 1/64 of the
                   inputs are +-inf, so that opposite infinities meet as NaN."""
    e_bits, m_bits, bias = FORMAT[dtype]
    rng = np.random.default_rng(0x10E0000 + seed)
    out = []
    for r in range(world):
        sign = rng.integers(0, 2, n)
        mant = rng.integers(0, 1 << m_bits, n)
        if kind == "full":
            lo, step, span, jitter = _FULL_BANDS[dtype]
            exp_field = bias + lo + (r * step) % span + rng.integers(0, jitter, n)
        elif kind == "subnormal":
            exp_field = rng.integers(0, 2, n)
        elif kind == "overflow":
            exp_field = np.full(n, (1 << e_bits) - 2)
            inf = rng.integers(0, 64, n) == 0
            exp_field[inf] = (1 << e_bits) - 1
            mant[inf] = 0
        else:
            raise ValueError(f"unknown kind {kind!r}")
        out.append(_from_fields(sign, exp_field, mant, dtype))
    if kind == "full" and world > 1:
        at = np.flatnonzero(rng.integers(0, 8, n) == 0)
        p = rng.integers(0, world, at.size)
        q = (p + 1 + rng.integers(0, world - 1, at.size)) % world
        big = _from_fields(np.zeros(at.size, np.int64), np.full(at.size, bias + _CANCEL_E[dtype]),
                           rng.integers(0, 1 << m_bits, at.size), dtype)
        for r in range(world):
            out[r][torch.from_numpy(at[p == r])] = big[torch.from_numpy(p == r)]
            out[r][torch.from_numpy(at[q == r])] = -big[torch.from_numpy(q == r)]
    return [v.to(device) for v in out]


def two_shot_expected(vas: List[torch.Tensor]) -> torch.Tensor:
    """VC of every rank after two-shot: slice s is fp32(VA[s]) + fp32(VA[s+1]) + ... (ranks mod P), rounded once."""
    world = len(vas)
    n = vas[0].numel()
    parts = []
    for s in range(world):
        seg = segment(n, world, s)
        acc = vas[s][seg].float()
        for q in range(1, world):
            acc = acc + vas[(s + q) % world][seg].float()
        parts.append(acc.to(vas[0].dtype))
    return torch.cat(parts)


def round16(x: np.ndarray, dtype: str, mode: str = "rne") -> torch.Tensor:
    """fp64 values rounded ONCE to the 16-bit type (``rne``: to nearest even, ``rz``: toward zero), computed exactly:
    the quantum of x's binade (or of the subnormal range) is a power of two, so x / quantum is exact and numpy rounds it
    to an integer.  Overflow past the largest finite value gives +-inf (``rne``) or the largest value (``rz``)."""
    e_bits, m_bits, bias = FORMAT[dtype]
    x = np.asarray(x, dtype=np.float64)
    _, e = np.frexp(x)                                      # x = m * 2^e, 0.5 <= |m| < 1
    q = np.ldexp(1.0, np.maximum(e, 2 - bias) - (m_bits + 1))
    r = (np.round(x / q) if mode == "rne" else np.trunc(x / q)) * q
    top = np.ldexp(1.0, (1 << e_bits) - 1 - bias)          # 2^(emax+1): the first value past the finite range
    big = np.abs(r) >= top
    if mode == "rne":
        r = np.where(big, np.copysign(np.inf, x), r)
    else:
        r = np.where(big, np.copysign(top - np.ldexp(top, -(m_bits + 1)), x), r)
    r = np.where(np.isnan(x), np.nan, r)
    return torch.from_numpy(r.astype(np.float32)).to(TORCH_DTYPE[dtype])   # exact: r has at most m_bits + 1 bits


def mismatches(got: torch.Tensor, want: torch.Tensor) -> int:
    """Elements whose bits differ, NaN compared by class (any NaN equals any NaN; -0.0 != 0.0)."""
    if got.shape != want.shape or got.dtype != want.dtype:
        raise ValueError(f"shape/dtype differ: {tuple(got.shape)} {got.dtype} vs {tuple(want.shape)} {want.dtype}")
    differ = bits(got) != bits(want)
    both_nan = torch.isnan(got) & torch.isnan(want)
    return int((differ & ~both_nan).sum())


def describe(got: torch.Tensor, want: torch.Tensor) -> str:
    """The first differing elements, for assertion messages."""
    differ = (bits(got) != bits(want)) & ~(torch.isnan(got) & torch.isnan(want))
    bad = differ.nonzero().flatten()[:4].tolist()
    return ", ".join(f"[{i} (vector {i // LANES})] got {got[i].item()!r} want {want[i].item()!r}" for i in bad)
