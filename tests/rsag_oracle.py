"""Expected results of the reduce-scatter + all-gather ring (ring_rsag_kernel, csrc/kernels/ring_allreduce.cu), bit for
bit, torch only; data and comparisons come from tests/allreduce_oracle.py.

The block of n elements is P segments of whole 16-byte vectors.  Segment s is summed once, by rank s, as
((VA[s+1] + VA[s+2]) + ...) + VA[s] (ranks mod P), one add at a time in the element type, so every rank ends with the
same bits:

* ``rsag_expected``           VC of every rank after the whole allreduce;
* ``reduce_scatter_expected`` segment s as rank s holds it after the reduce-scatter half (the rest of VC is untouched);
* ``all_gather_expected``     VC of every rank after the all-gather half alone: segment s is rank s's VA[s].
"""
from __future__ import annotations

from typing import List

import torch


def segment(n: int, world: int, s: int) -> slice:
    """Elements of segment ``s`` (``n`` is a multiple of world 16-byte vectors)."""
    return slice(s * n // world, (s + 1) * n // world)


def reduce_scatter_expected(vas: List[torch.Tensor], s: int) -> torch.Tensor:
    """Segment ``s`` as rank ``s`` sums it: ((VA[s+1] + VA[s+2]) + ...) + VA[s], one add at a time."""
    world = len(vas)
    seg = segment(vas[0].numel(), world, s)
    acc = vas[(s + 1) % world][seg].clone()
    for k in range(2, world + 1):
        acc = acc + vas[(s + k) % world][seg]
    return acc


def rsag_expected(vas: List[torch.Tensor]) -> torch.Tensor:
    """VC of every rank after the reduce-scatter + all-gather ring (every rank holds the same bits)."""
    return torch.cat([reduce_scatter_expected(vas, s) for s in range(len(vas))])


def all_gather_expected(vas: List[torch.Tensor]) -> torch.Tensor:
    """VC of every rank after the all-gather phase alone: segment s is rank s's VA[s]."""
    world = len(vas)
    return torch.cat([vas[s][segment(vas[0].numel(), world, s)] for s in range(world)])
