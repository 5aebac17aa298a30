"""Element-wise oracle of the allreduce kernels (csrc/kernels/ring_allreduce.cu): data and expected results, torch only.

The miniapps check the reference's way: rank r holds the constant r, every element of VC must equal P(P-1)/2.  That
check cannot see a chunk added at the wrong place, a slot read one launch too early, a carry lost between lanes or a
changed summation order.  The data here varies per rank, per element and per launch, and the expected values are
computed operation by operation in the element type:

* ``make_inputs``     one VA per rank; integers over their full range (sums wrap, carries cross every byte and 32-bit
                      boundary), floats from a normal distribution, or integer-valued floats in +-2^20 (``exact``:
                      every partial sum of at most 16 of them, the most ranks a kernel takes, is exact in any order);
* ``ring_expected``   VC of the fused ring (push and pull, both slot policies) and of the unfused ring, bit for bit:
                      rank r adds VA[r], VA[r-1], ..., VA[r-P+1] into a zeroed VC, one add at a time;
* ``allreduce_bound`` the fp64 sum and the error bound of recursive summation in any order, for two-shot, whose
                      order differs between its main blocks (owner first) and its tail loop (rank 0 first);
* ``two_shot_sum_pinned`` two-shot's float and double sum in exactly the kernel's order (main blocks owner first, tail
                      vectors rank 0 first, the boundary from ``TWO_SHOT_SHAPES``), bit for bit;
* ``mismatches`` / ``two_shot_problems`` the comparisons the GPU tests assert on.
"""
from __future__ import annotations

from typing import List, Tuple

import torch

DTYPES = ("float", "int", "uint", "double", "long", "ulong", "short", "ushort", "uchar")
FLOATING = ("float", "double")
# reference element type -> the torch dtype whose add is bit-identical (unsigned integers share the two's-complement
# add of the signed type of the same width)
TORCH_DTYPE = {"float": torch.float32, "int": torch.int32, "uint": torch.int32, "double": torch.float64,
               "long": torch.int64, "ulong": torch.int64, "short": torch.int16, "ushort": torch.int16,
               "uchar": torch.uint8}
EXACT_RANGE = 1 << 20
MAX_RANKS = 16              # kApiMaxRanks (csrc/kernels/api.h)
_BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
# Two-shot's <W, U> by world size (kTwoShotShapes, csrc/kernels/ring_allreduce.cuh): the first row with world <= W runs.
# Every launch has 512 threads per CTA, and a CTA reduces 512 * U vectors per trip of the main loop.
TWO_SHOT_SHAPES = ((2, 4), (4, 4), (8, 2), (16, 1))
TWO_SHOT_THREADS = 512


def two_shot_u(world: int) -> int:
    """U of the two-shot kernel that runs at ``world`` ranks."""
    return next(u for w, u in TWO_SHOT_SHAPES if world <= w)


def two_shot_main_vectors(slice_vec: int, world: int, u: int = 0) -> int:
    """Vectors of a slice of ``slice_vec`` that the main blocks reduce; the tail loop takes the rest (``u`` overrides
    the kernel's U)."""
    block = TWO_SHOT_THREADS * (u or two_shot_u(world))
    return slice_vec // block * block


def elem_bytes(dtype: str) -> int:
    return torch.empty((), dtype=TORCH_DTYPE[dtype]).element_size()


def lanes(dtype: str) -> int:
    """Elements per 16-byte vector, the unit every allreduce kernel moves and adds."""
    return 16 // elem_bytes(dtype)


def make_inputs(world: int, n: int, dtype: str, seed: int, exact: bool = False,
                device: str = "cpu") -> List[torch.Tensor]:
    """VA of every rank (``n`` elements each), different per rank, per element and per ``seed``."""
    td = TORCH_DTYPE[dtype]
    g = torch.Generator(device=device).manual_seed(0x5EED0000 + seed)
    out = []
    for _ in range(world):
        if dtype not in FLOATING:
            raw = torch.randint(0, 256, (n * elem_bytes(dtype),), dtype=torch.uint8, generator=g, device=device)
            out.append(raw.view(td))
        elif exact:
            out.append(torch.randint(-EXACT_RANGE, EXACT_RANGE + 1, (n,), generator=g, device=device).to(td))
        else:
            out.append(torch.randn(n, dtype=td, generator=g, device=device))
    return out


def ring_expected(vas: List[torch.Tensor], rank: int) -> torch.Tensor:
    """VC of ``rank`` after the ring: 0 + VA[rank] + VA[rank-1] + ... + VA[rank-P+1], one add at a time."""
    world = len(vas)
    acc = torch.zeros_like(vas[0])
    for t in range(world):
        acc = acc + vas[(rank - t) % world]
    return acc


def allreduce_bound(vas: List[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(fp64 sum, bound): any recursive summation of the P blocks in the element type lies within ``bound`` of the sum.

    Recursive summation of P terms errs by at most gamma_{P-1} * sum|x| with gamma_k = k*u / (1 - k*u), u the unit
    roundoff of the element type; the fp64 sum itself errs by at most (P-1) * 2^-53 * sum|x| (it is exact for fp32
    inputs in all but extreme exponent spreads, not for fp64 ones), so both terms enter the bound."""
    world = len(vas)
    x = torch.stack([v.to(torch.float64) for v in vas])
    u = torch.finfo(vas[0].dtype).eps / 2
    k = world - 1
    gamma = k * u / (1 - k * u) + k * 2.0 ** -53
    return x.sum(0), gamma * x.abs().sum(0)


def two_shot_sum_pinned(vas: List[torch.Tensor], u: int = 0) -> torch.Tensor:
    """VC of every rank after a float or double two-shot sum, in the kernel's order: within slice s, the main-block
    vectors add owner first, ((VA[s] + VA[s+1]) + ...) + VA[s+P-1] (ranks mod P), and the tail vectors rank 0 first,
    ((VA[0] + VA[1]) + ...) + VA[P-1], one IEEE add at a time.  ``u`` overrides the kernel's U."""
    world, n = len(vas), vas[0].numel()
    if vas[0].dtype not in (torch.float32, torch.float64):
        raise ValueError(f"the pinned order is the float and double sum's, not {vas[0].dtype}'s")
    per, per_vec = n // world, 16 // vas[0].element_size()
    main = two_shot_main_vectors(per // per_vec, world, u) * per_vec
    out = []
    for s in range(world):
        lo = s * per
        head = vas[s][lo:lo + main].clone()
        for q in range(1, world):
            head = head + vas[(s + q) % world][lo:lo + main]
        tail = vas[0][lo + main:lo + per].clone()
        for p in range(1, world):
            tail = tail + vas[p][lo + main:lo + per]
        out += [head, tail]
    return torch.cat(out)


def bits(t: torch.Tensor) -> torch.Tensor:
    """The raw bits of every element (so that -0.0 != 0.0 and NaN == NaN of the same payload)."""
    return t.view(_BITS[t.element_size()])


def mismatches(got: torch.Tensor, want: torch.Tensor) -> int:
    """Elements whose bits differ."""
    if got.shape != want.shape or got.dtype != want.dtype:
        raise ValueError(f"shape/dtype differ: {tuple(got.shape)} {got.dtype} vs {tuple(want.shape)} {want.dtype}")
    return int((bits(got) != bits(want)).sum())


def describe(got: torch.Tensor, want: torch.Tensor, lanes_per_vec: int = 1) -> str:
    """The first differing elements, for assertion messages."""
    bad = (bits(got) != bits(want)).nonzero().flatten()[:4].tolist()
    return ", ".join(f"[{i} (vector {i // lanes_per_vec})] got {got[i].item()!r} want {want[i].item()!r}" for i in bad)


def two_shot_problems(vcs: List[torch.Tensor], vas: List[torch.Tensor], exact: bool) -> List[str]:
    """What is wrong with the VC of every rank after a two-shot allreduce of ``vas`` ([] = nothing).

    Every rank must hold the same bits (each slice is reduced once, by its owner, and stored to every rank).  Exact
    data (integers, or ``exact`` floats) must equal the sum bit for bit; random floats must lie within
    ``allreduce_bound`` (the order of the adds is not uniform across a slice, so no one order is pinned)."""
    problems = []
    for r in range(1, len(vcs)):
        k = mismatches(vcs[r], vcs[0])
        if k:
            problems.append(f"rank {r} differs from rank 0 in {k} elements: {describe(vcs[r], vcs[0])}")
    if exact or vas[0].dtype not in (torch.float32, torch.float64):
        want = ring_expected(vas, 0)
        k = mismatches(vcs[0], want)
        if k:
            problems.append(f"{k} elements differ from the exact sum: {describe(vcs[0], want)}")
    else:
        ref, bound = allreduce_bound(vas)
        err = (vcs[0].to(torch.float64) - ref).abs()
        bad = ~(err <= bound)                   # NaN is out of bounds too
        if bool(bad.any()):
            i = int(bad.nonzero()[0])
            problems.append(f"{int(bad.sum())} elements outside the summation bound, first [{i}]: "
                            f"got {vcs[0][i].item()!r}, sum {ref[i].item()!r}, bound {bound[i].item()!r}")
    return problems
