"""The collectives that end in the node barrier at 9 to 16 ranks on one H100, bit for bit, on serial ranks.

Above 8 virtual ranks the concurrent drivers cannot run (``VirtualRanks.MAX_WORLD``: the spinning grids of two ranks
that share one of the device's hardware queues serialise, and the barrier times out).  tests/wide_world.py runs the P
launches one after another on ONE stream with pre-armed barrier words instead, so every world from 9 to 16 runs on one
GPU: the 16-wide bucket of kTwoShotShapes ({16, 1}) of ``two_shot_kernel``, ``two_shot_f32_kernel``,
``reduce_scatter_kernel`` and ``reduce_scatter_f32_kernel``, which no smaller world takes, and the ``q < world`` guards,
``(rank + q) % world`` walks, barrier words 8..15 and the all-to-all-v's judges at rows and columns 8..15 of the shared
kernels.  Every case runs three launches with fresh data and an advancing epoch; every output starts poisoned, inputs
must come back unchanged, and after every launch each rank's arrival word, status word and ticket word are exact.

* two-shot allreduce: all 96 (type, op) pairs the binding takes at 9 and 16 ranks, the float and int sums at every world
  from 9 to 16, and slices of 37 vectors (tail only), 512 (exactly one U = 1 block) and 3 * 512 + 1 (blocks and a tail)
  with 1 CTA, 3 CTAs and the default grid; float and double sums against the kernel's pinned order;
* reduce-scatter: the same 96 pairs at 9, 12 and 16 ranks with segments of one vector and of 2085 (four U = 1 blocks and
  a 37-vector tail), and float and double sums over 4 MiB segments at 16 ranks (1 GiB of send buffers);
* all-to-all and all-gather, push and pull, at 9, 13 and 16 ranks with blocks of 16 B, 48 B, 4 KiB + 16 B and 1 MiB;
* all-to-all-v, push and pull, at 9 and 16 ranks with rows of 16 B, 48 B and 4 KiB + 16 B: every count pattern of
  tests/alltoallv_oracle.py, then one refused matrix per rule with its bad entry in the last row or column, each moving no
  byte with the same verdict on every rank, and a valid launch after each.

The value-index pair types run one U = 1 block and a 37-vector tail instead of the larger sizes, and their reduce-scatter
runs it at 16 ranks only: their oracle folds one pair at a time in Python.
"""
import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
import tests.bitop_oracle as bit
import tests.loc_oracle as loc
import tests.reduce_op_oracle as rop
import tests.wide_world as ww
from tests.alltoallv_oracle import PATTERNS, RECV_CAPACITY, NEGATIVE, SEND_CAPACITY, counts_for

pytestmark = pytest.mark.gpu

DEV = 0
CASES = ([(t, op) for t in rop.TYPES for op in ("sum",) + rop.OPS]
         + [(t, op) for t in bit.INT_TYPES for op in bit.BIT_OPS]
         + [(t, op) for t in loc.PAIR_TYPES for op in loc.LOC_OPS])
IDS = [f"{t}-{o}" for t, o in CASES]
BLOCK = 512                 # vectors of one main block at U = 1 (kTwoShotShapes {16, 1}, 512 threads)
TAIL_VEC = 4 * BLOCK + 37   # four main blocks and a 37-vector tail
PAIR_VEC = BLOCK + 37       # the pair types' larger size


@pytest.fixture
def serial():
    made = []

    def make(world):
        made.append(ww.SerialRanks(world, DEV))
        return made[-1]

    yield make
    for sr in made:
        sr.close()


# ---------------------------------------------------------------------------------------------------------- two-shot ----
@pytest.mark.parametrize("world", [9, 16])
@pytest.mark.parametrize("dtype,op", CASES, ids=IDS)
def test_two_shot_every_type_and_op(serial, dtype, op, world):
    ww.two_shot(serial(world), dtype, op, PAIR_VEC if dtype in loc.PAIR_TYPES else 3 * BLOCK + 1)


@pytest.mark.parametrize("dtype", ["float", "int"])
@pytest.mark.parametrize("world", range(9, 17))
def test_two_shot_sums_at_every_world(serial, world, dtype):
    ww.two_shot(serial(world), dtype, "sum", 3 * BLOCK + 1)


@pytest.mark.parametrize("ctas", [1, 3, 0], ids=["1cta", "3ctas", "default"])
@pytest.mark.parametrize("slice_vec", [37, BLOCK, 3 * BLOCK + 1], ids=["tail-only", "one-block", "blocks+tail"])
@pytest.mark.parametrize("world", [9, 16])
@pytest.mark.parametrize("dtype", ["float", "double"])
def test_two_shot_pinned_sum_slices_and_grids(serial, dtype, world, slice_vec, ctas):
    ww.two_shot(serial(world), dtype, "sum", slice_vec, ctas=ctas)


# ---------------------------------------------------------------------------------------------------- reduce-scatter ----
# The pair types' Python oracle is slow: their blocks-and-tail segment runs at 16 ranks only.
RS = [(t, op, world, seg) for t, op in CASES for world in (9, 12, 16) for seg in (1, TAIL_VEC)
      if t not in loc.PAIR_TYPES or seg == 1 or world == 16]


@pytest.mark.parametrize("dtype,op,world,seg_vec", RS, ids=[f"{t}-{o}-{w}-{v}v" for t, o, w, v in RS])
def test_reduce_scatter_every_type_and_op(serial, dtype, op, world, seg_vec):
    ww.reduce_scatter(serial(world), dtype, op, PAIR_VEC if dtype in loc.PAIR_TYPES and seg_vec > 1 else seg_vec)


@pytest.mark.parametrize("dtype", ["float", "double"])
def test_reduce_scatter_4_mib_segments(serial, dtype):
    ww.reduce_scatter(serial(16), dtype, "sum", (4 << 20) // 16)


# ------------------------------------------------------------------------------------------ all-to-all, all-gather ----
BLOCKS = [16, 48, 4096 + 16, 1 << 20]


@pytest.mark.parametrize("pull", [False, True], ids=["push", "pull"])
@pytest.mark.parametrize("block_bytes", BLOCKS, ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [9, 13, 16])
def test_all_to_all(serial, world, block_bytes, pull):
    ww.all_to_all(serial(world), block_bytes, pull)


@pytest.mark.parametrize("pull", [False, True], ids=["push", "pull"])
@pytest.mark.parametrize("block_bytes", BLOCKS, ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [9, 13, 16])
def test_all_gather(serial, world, block_bytes, pull):
    ww.all_gather(serial(world), block_bytes, pull)


# ---------------------------------------------------------------------------------------------------- all-to-all-v ----
@pytest.mark.parametrize("pull", [False, True], ids=["push", "pull"])
@pytest.mark.parametrize("row_bytes", [16, 48, 4096 + 16], ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [9, 16])
def test_all_to_all_v(serial, world, row_bytes, pull):
    sr = serial(world)
    v = ww.AllToAllV(sr, row_bytes, pull)
    gen = torch.Generator().manual_seed(world + row_bytes)
    for pattern in PATTERNS:
        for launch in range(ww.LAUNCHES):
            v.launch(counts_for(pattern, world, ww.MEAN, v.cap, launch, gen), launch, seed=len(pattern))
    for rule in (NEGATIVE, SEND_CAPACITY, RECV_CAPACITY):
        v.launch(v.refused(rule), 0, seed=rule)           # no byte moves, every rank says `rule`
        v.launch(counts_for("random", world, ww.MEAN, v.cap, rule, gen), 1, seed=rule)
    assert sr.epoch == len(PATTERNS) * ww.LAUNCHES + 6
