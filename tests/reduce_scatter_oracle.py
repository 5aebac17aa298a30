"""Exact reference of the stand-alone reduce-scatter (csrc/kernels/api.h: launch_reduce_scatter), built on the
allreduce oracles.

Rank p's send buffer holds P segments of n elements; rank r's result is the owner-first fold of segment r,
((S_r[r] o S_{r+1}[r]) o ...) o S_{r+P-1}[r] (ranks mod P), in every element, the tail included:
  sum          one add at a time in the type (integers wrap); bfloat16 / half in fp32, rounded once
  prod / min / max           tests/reduce_op_oracle.py's combine (16-bit prod in fp32, rounded once)
  band ... lxor              tests/bitop_oracle.py's fold (one part: itself, unnormalised)
  maxloc / minloc            tests/loc_oracle.py's combine, padding zero (one part: its bytes as they are)
"""
from typing import List

import numpy as np
import torch

import tests.bitop_oracle as bit
import tests.loc_oracle as loc
import tests.reduce_op_oracle as rop

LOWP = ("bfloat16", "half")


def _segments(t: torch.Tensor, world: int) -> List[torch.Tensor]:
    return list(t.reshape(world, -1))


def expected(sends, r: int, op: str, dtype: str):
    """Rank r's receive buffer: a tensor of the dtype's torch type, or bytes for a pair type (``sends[p]`` then holds
    rank p's send buffer as bytes)."""
    world = len(sends)
    order = [(r + k) % world for k in range(world)]
    if dtype in loc.PAIR_TYPES:
        seg = len(sends[0]) // world
        return fold([sends[p][r * seg:(r + 1) * seg] for p in order], op, dtype)
    return fold([_segments(sends[p], world)[r] for p in order], op, dtype)


def fold(segs, op: str, dtype: str):
    """((segs[0] o segs[1]) o ...) element by element, in the kernels' arithmetic (the module docstring): tensors of the
    dtype's torch type, or bytes for a pair type.  One part comes back as it is."""
    if dtype in loc.PAIR_TYPES:
        if len(segs) == 1:
            return bytes(segs[0])
        parts = [loc.unpack_all(s, dtype) for s in segs]
        out = []
        for k in range(len(parts[0])):
            acc = parts[0][k]
            for part in parts[1:]:
                acc = loc.combine(op, acc, part[k])
            out.append(loc.pack_result(acc, dtype))
        return b"".join(out)
    if op == "sum":
        if dtype in LOWP:
            acc = segs[0].float()
            for x in segs[1:]:
                acc = acc + x.float()
            return acc.to(segs[0].dtype)
        bits = [rop.to_bits(x) for x in segs]
        vals = [rop.values(b, dtype) for b in bits]
        acc = vals[0].copy()
        with np.errstate(all="ignore"):
            for v in vals[1:]:
                acc = acc + v                      # IEEE add in the type, or wrapping integer add
        return torch.from_numpy(np.ascontiguousarray(acc)).view(rop.TORCH_DTYPE[dtype]) \
            if dtype not in ("uint", "ulong", "ushort") else rop.from_bits(acc.view(bits[0].dtype), dtype)
    if op in bit.BIT_OPS:
        return rop.from_bits(bit.fold([rop.to_bits(x) for x in segs], op, dtype), dtype)
    parts = [rop.to_bits(x) for x in segs]
    if op == "prod" and dtype in LOWP:
        return rop.from_bits(rop._prod16_f32(parts, dtype), dtype)
    return rop.from_bits(rop._fold(parts, op, dtype), dtype)


def make_inputs(world: int, n: int, dtype: str, op: str, seed: int, launch: int):
    """Every rank's send buffer (P segments of n elements) with the adversarial inputs of the oracle that owns (op,
    dtype): NaN, +-0, subnormals, wraparound, loc ties and garbage padding; the sum gets random finite values."""
    total = world * n
    if dtype in loc.PAIR_TYPES:
        kind = loc.KINDS[launch % len(loc.KINDS)]
        return loc.make_inputs(world, total, dtype, seed + launch, kind, garbage_padding=True)
    if op in bit.BIT_OPS:
        return bit.make_inputs(world, total, dtype, seed + launch, bit.KINDS[launch % len(bit.KINDS)])
    if op == "sum":
        import tests.allreduce_oracle as aro
        import tests.lowp_allreduce_oracle as lowp
        if dtype in LOWP:
            return lowp.make_inputs(world, total, dtype, seed + launch)
        return aro.make_inputs(world, total, dtype, seed + launch)
    k = rop.kinds(op, dtype)
    return rop.make_inputs(world, total, dtype, seed=seed + launch, op=op, kind=k[launch % len(k)])


def bits_equal(got, want, dtype: str) -> int:
    """Elements whose bits differ (pair types: differing pairs, padding included)."""
    if dtype in loc.PAIR_TYPES:
        return loc.mismatches(got, want, dtype)
    return rop.mismatches(got, want)
