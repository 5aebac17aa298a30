"""The data of the tensor-parallel layer tests (tests/tp_oracle.py) and the exact MLP construction, on the CPU.

A layer that reuses last step's rows, weights or sums, or hands one rank's result to another, must fail the GPU tests
(test_gpu_tensor_parallel.py), so the expected results of consecutive steps and of different ranks must differ almost
everywhere; the exact MLP case must be exact in fp32 whatever order the two GEMMs add in."""
import numpy as np
import pytest
import torch

from tests.gemm_oracle import FP32_BITS, SILU_OVERFLOW, mlp_down_bits, mlp_exact_operands, reference, rne_bf16, round_bits
from tests.tp_oracle import (COLUMN_CASES, MLP_CASES, MLP_STEPS, ROW_CASES, STEPS, column_step, fraction_differing,
                             mlp_hidden, mlp_output, mlp_step, row_expected, row_step)

DIFFER = 0.99


def _distinct(outputs):
    """outputs[step][rank]: consecutive steps and every pair of ranks differ in >= 99 % of the elements."""
    for s in range(1, len(outputs)):
        for r, (now, before) in enumerate(zip(outputs[s], outputs[s - 1])):
            f = fraction_differing(now, before)
            assert f >= DIFFER, f"step {s} rank {r}: only {f:.4f} of the elements differ from step {s - 1}"
    for s, per_rank in enumerate(outputs):
        for q in range(1, len(per_rank)):
            for r in range(q):
                f = fraction_differing(per_rank[q], per_rank[r])
                assert f >= DIFFER, f"step {s}: ranks {r} and {q} differ in only {f:.4f} of the elements"


@pytest.mark.parametrize("case", ROW_CASES, ids=str)
def test_row_parallel_data_differs_per_step_and_rank(case):
    _distinct([row_expected(row_step(case, s)[2], case.world) for s in range(STEPS)])


@pytest.mark.parametrize("case", COLUMN_CASES, ids=str)
def test_column_parallel_data_differs_per_step_and_rank(case):
    """On C before the activation (relu zeroes half of it on every step), and on the gathered rows themselves."""
    steps = [column_step(case, s) for s in range(STEPS)]
    _distinct([c for _, _, _, c in steps])
    _distinct([xs for xs, _, _, _ in steps])
    for _, _, _, cs in steps:
        assert all(float(c.min()) < SILU_OVERFLOW < 87 < float(c.max()) for c in cs)     # past silu's overflow


@pytest.mark.parametrize("case", MLP_CASES, ids=str)
def test_mlp_data_differs_per_step_and_rank_and_stays_normal(case):
    steps = [mlp_step(case, s) for s in range(MLP_STEPS)]
    _distinct([cs for _, _, _, cs in steps])
    outs = []
    for _, _, w_downs, cs in steps:
        assert case.exact or all(float(c.abs().max()) < 80 for c in cs)  # silu(C) and gelu(C) stay normal
        hs = [mlp_hidden(c, case.activation) for c in cs]
        nz = torch.cat([h.double().abs().flatten() for h in hs])
        assert float(nz[nz > 0].min()) >= 2.0 ** -100
        y, _ = mlp_output(hs, w_downs, case.world)
        outs.append(y)
        assert all(float(v[v != 0].abs().min()) >= 2.0 ** -100 for v in y)
    _distinct(outs)


# ---- the exact MLP construction ------------------------------------------------------------------------------------
def test_mlp_exact_budget():
    assert mlp_down_bits(256, 512, 2, 3) == FP32_BITS                  # the GPU test's exact case uses all 24 bits
    assert mlp_down_bits(256, 256, 2, 3) == 23
    with pytest.raises(ValueError):
        mlp_exact_operands(256, 256, 512, 0, p_down=4)
    with pytest.raises(ValueError):
        mlp_exact_operands(256, 256, 1024, 0)


def test_mlp_exact_operands_have_the_stated_form():
    x, w_up, w_down = mlp_exact_operands(256, 256, 512, seed=3)
    for t, p in ((x, 2), (w_up, 2), (w_down, 3)):
        t64 = t.double()
        assert torch.equal(round_bits(t64, p), t64) and bool((round_bits(t64, p - 1) != t64).any())
        e = torch.frexp(t64)[1]
        assert bool((e == e[:, :1]).all())                             # one exponent per row, over all ranks' blocks
    assert int(torch.frexp(w_up.double())[1].max()) == int(torch.frexp(w_up.double())[1].min()) == 1   # 2^0


@pytest.mark.parametrize("world", [1, 2])
def test_mlp_exact_under_fp32_accumulation_in_any_order(world):
    """Both GEMMs of the exact case, emulated in numpy fp32: the first in random orders (h is then rne_bf16(relu(C))
    exactly), the second per rank in random orders and then the P shard additions in random orders, for 24 rows x
    32 columns of every rank's output: always the fp64 product of the hidden values."""
    tokens, hidden, ffn = 128 * world * 2, 256, 256 * world * (2 if world == 1 else 1)
    x, w_up, w_down = mlp_exact_operands(tokens, hidden, ffn, seed=10 + world)
    rows = torch.arange(0, tokens, tokens // 24)[:24]
    c = reference(x, w_up)
    h = rne_bf16(c.clamp(min=0))
    assert float((h.double() == 0).double().mean()) < 0.6
    assert bool((h.double() != c.clamp(min=0)).any())                  # some hidden values are rounded
    rng = np.random.default_rng(world)
    up_terms = (x.float()[rows, None, :] * w_up.float()[None, :64, :]).numpy()
    for order in [np.arange(hidden)] + [rng.permutation(hidden) for _ in range(2)]:
        acc = np.zeros(up_terms.shape[:2], dtype=np.float32)
        for i in order:
            acc += up_terms[:, :, i]
        assert np.array_equal(acc.astype(np.float64), c[rows, :64].numpy())
    want = reference(h, w_down)[rows, :32].numpy()
    terms = (h.float()[rows, None, :] * w_down.float()[None, :32, :]).numpy()     # bf16 x bf16: exact in fp32
    k_local = ffn // world
    for _ in range(3):
        partials = []
        for r in range(world):
            acc = np.zeros(terms.shape[:2], dtype=np.float32)
            for i in r * k_local + rng.permutation(k_local):
                acc += terms[:, :, i]
            partials.append(acc)
        shard = np.zeros_like(partials[0])
        for r in rng.permutation(world):
            shard += partials[r]
        assert np.array_equal(shard.astype(np.float64), want)
