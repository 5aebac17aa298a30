"""Cases, data and expected values of the tensor-parallel layer tests (test_gpu_tensor_parallel.py), torch only.

Every step of every case draws new activations AND new weights for every rank from ``tests/gemm_oracle.py``, so a layer
that computes with last step's rows, weights or sums fails; test_tp_oracle.py asserts on the CPU that the expected
results of consecutive steps, and of different ranks, differ almost everywhere.

* ``row_step``     ``RowParallelLinear``: one ``exact_operands`` product with world * K_local terms, cut into the ranks'
                   K-slices (one exponent per row over all ranks, so the sum over ranks is exact in fp32 in any order).
* ``column_step``  ``ColumnParallelLinear``: the gathered A and one weight per rank, |C| past silu's overflow point.
* ``mlp_step``     ``ParallelMLP``: ``mlp_exact_operands`` for the exact case, else full-mantissa data with |C| of the
                   first GEMM below 80, so that every hidden value and every term of the second GEMM stays normal.
"""
from __future__ import annotations

import math
import zlib
from typing import List, NamedTuple

import torch

from tests.gemm_oracle import activation64, exact_operands, mantissa_bits, mlp_exact_operands, reference, rne_bf16

MAX = "max"            # ctas: the co-resident maximum, every rank's grid resident at once
STEPS = 4


class RowCase(NamedTuple):
    world: int
    tiles: int         # 128-row tiles per shard: M = 128 * world * tiles (2 for CTA pairs: cluster=2 needs even)
    nb: int            # N / 256
    kb: int            # K_local / 64
    cluster: int
    ctas: object       # MAX or a number of CTAs (several tiles per CTA)
    variant: str       # red | tma (fp32 shards) | bf16

    @property
    def shape(self):
        return 128 * self.world * self.tiles, 256 * self.nb, 64 * self.kb


ROW_CASES = [RowCase(*c) for c in [
    (1, 1, 3, 64, 0, MAX, "red"), (1, 3, 1, 1, 1, 3, "tma"), (1, 2, 1, 3, 2, MAX, "bf16"),
    (2, 3, 1, 3, 1, MAX, "red"), (2, 2, 3, 1, 2, 3, "tma"), (2, 1, 1, 64, 0, 1, "bf16"),
    (3, 1, 1, 1, 0, 3, "red"), (3, 2, 1, 64, 2, MAX, "tma"), (3, 3, 3, 3, 1, MAX, "bf16"),
    (4, 2, 1, 3, 2, MAX, "red"), (4, 1, 3, 1, 1, MAX, "tma"), (4, 3, 1, 3, 0, 3, "bf16"),
    (5, 3, 3, 1, 1, 1, "red"), (5, 1, 1, 3, 0, MAX, "tma"), (5, 2, 3, 1, 2, MAX, "bf16"),
    (8, 1, 1, 64, 1, MAX, "red"), (8, 2, 1, 1, 2, 3, "tma"), (8, 3, 1, 3, 0, MAX, "bf16"),
]]


class ColumnCase(NamedTuple):
    world: int
    chunk: int         # gather granularity in bytes (0: the default, 4096)
    activation: str
    ctas: object
    cluster: int

    @property
    def shape(self):
        rows = 128 * (2 if self.world <= 3 else 1)
        return rows * self.world, 256 * (1 + self.world % 2), 256      # M, N_local, K


ACTIVATIONS = ["none", "relu", "gelu", "silu"]
CHUNKS = [0, 512, 2048, 4096]
# cluster 0 (CTA pairs where the shard allows them) only on small grids: a partly resident pair grid could wait for a
# CTA of another rank's kernel that cannot start.
COLUMN_CASES = [ColumnCase(w, CHUNKS[(w + i) % 4], act, MAX if (w + i) % 2 else 3, 1 if (w + i) % 2 else 0)
                for w in range(1, 9) for i, act in enumerate(ACTIVATIONS)]


class MlpCase(NamedTuple):
    world: int
    activation: str
    exact: bool        # mlp_exact_operands data: the block output bit for bit
    ctas: object

    @property
    def shape(self):
        return 128 * self.world * (2 if self.exact else 1), 256, 256 * self.world    # tokens, hidden, ffn


MLP_CASES = [MlpCase(2, "relu", True, MAX)] + [MlpCase(w, act, False, MAX if i % 2 == 0 else 3)
                                              for w in (1, 2, 4, 8) for i, act in enumerate(["relu", "gelu", "silu"])]
MLP_STEPS = 3
ACT_EXP = dict(a_exp=(-10, 2), b_exp=(-3, 0))      # |C| from below 2^-8 to ~150 at K = 256: past silu's -87
MLP_EXP = dict(a_exp=(-8, -3), b_exp=(-3, 0))      # |C| below 80 at hidden = 256 (asserted in test_tp_oracle.py)


def _seed(case, step: int) -> int:
    return (zlib.crc32(repr(tuple(case)).encode()) & 0xFFFFF) * 16 + step


def _blocks(t: torch.Tensor, world: int, dim: int) -> List[torch.Tensor]:
    return [c.contiguous() for c in t.chunk(world, dim)]


# The data is drawn on the CPU (the same values on every device) and moved to ``device``, where the references are
# computed.
# ---- RowParallelLinear ---------------------------------------------------------------------------------------------
def row_step(case: RowCase, step: int, device="cpu"):
    """(x_r, w_r per rank, fp64 partial products of every rank [M, N])."""
    m, n, k = case.shape
    extra = math.ceil(math.log2(case.world))
    a, b = exact_operands(m, n, case.world * k, _seed(case, step), p=mantissa_bits(k, extra))
    xs, ws = _blocks(a.to(device), case.world, 1), _blocks(b.to(device), case.world, 1)
    return xs, ws, [reference(x, w) for x, w in zip(xs, ws)]


def row_expected(partials: List[torch.Tensor], world: int) -> List[torch.Tensor]:
    """fp64 rows of the sum over ranks that rank r's shard holds."""
    return list(sum(partials).chunk(world, 0))


# ---- ColumnParallelLinear ------------------------------------------------------------------------------------------
def column_step(case: ColumnCase, step: int, device="cpu"):
    """(x_r rows per rank, w_r per rank, the gathered A, fp64 C_r = A @ w_r^T per rank, before the activation)."""
    m, n, k = case.shape
    seed = _seed(case, step)
    a = exact_operands(m, 256, k, seed, **ACT_EXP)[0].to(device)
    ws = [exact_operands(256, n, k, seed * 31 + 1 + r, **ACT_EXP)[1].to(device) for r in range(case.world)]
    return _blocks(a, case.world, 0), ws, a, [reference(a, w) for w in ws]


# ---- ParallelMLP ---------------------------------------------------------------------------------------------------
def mlp_step(case: MlpCase, step: int, device="cpu"):
    """(x rows, w_up row block, w_down column block per rank; fp64 C_r of the first GEMM per rank)."""
    tokens, hidden, ffn = case.shape
    seed = _seed(case, step)
    if case.exact:
        x, w_up, w_down = mlp_exact_operands(tokens, hidden, ffn, seed)
    else:
        x, w_up = exact_operands(tokens, ffn, hidden, seed, **MLP_EXP)
        w_down = exact_operands(hidden, 256, ffn, seed + 7, a_exp=(-3, 0))[0]
    x, w_up, w_down = x.to(device), w_up.to(device), w_down.to(device)
    ups = _blocks(w_up, case.world, 0)
    return _blocks(x, case.world, 0), ups, _blocks(w_down, case.world, 1), [reference(x, w) for w in ups]


def mlp_hidden(c: torch.Tensor, activation: str) -> torch.Tensor:
    """The bf16 hidden values of an exact epilogue: the fp64 activation of the exact C, rounded once."""
    return rne_bf16(activation64(c, activation))


def mlp_output(hs: List[torch.Tensor], w_downs: List[torch.Tensor], world: int):
    """(fp64 block output rows of every rank, the matching rows of sum_r |h_r| |w_down_r|^T) from hidden values."""
    full = sum(reference(h, w) for h, w in zip(hs, w_downs))
    mag = sum(h.double().abs() @ w.double().abs().t() for h, w in zip(hs, w_downs))
    return list(full.chunk(world, 0)), list(mag.chunk(world, 0))


def fraction_differing(x: torch.Tensor, y: torch.Tensor) -> float:
    return float((x.double() != y.double()).double().mean())
