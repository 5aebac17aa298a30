"""The GEMM oracle (tests/gemm_oracle.py) against emulated faulty kernels, on the CPU.

Each fault below is a way the wgmma GEMM kernels could lose precision or misplace data.  It is applied to a correct
result of a 128 x 256 x K product, and the comparison the GPU tests assert with (test_gpu_gemm_numerics.py) must report
it on the oracle's exact full-mantissa data.  Where the small dyadic data of the older GEMM tests hides the fault, that
is asserted too: it is the gap the exact data closes.  The construction itself is checked first: every value is a bf16
value with the stated number of bits, and the product is exact under fp32 accumulation in any order and under a model
of a tensor-core adder that aligns each 16-term block to its largest addend and keeps a 24-bit window."""
import itertools

import numpy as np
import pytest
import torch

from tests.gemm_oracle import (activation64, activation_bound, bf16_shard_outcomes, dyadic_operands, exact_operands,
                               general_bound, mantissa_bits, mismatches, reference, rne_bf16, round_bits,
                               shard_problems)

M, N, KB = 128, 256, 64
KS = (64, 256, 1024, 4096)


def _exact(k, seed=1, **kw):
    return exact_operands(M, N, k, seed, **kw)


def _blocked(a, b, hold):
    """The k-block loop of the kernel with the accumulator passed through ``hold`` after every 64-deep block."""
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float64)
    for k0 in range(0, a.shape[1], KB):
        acc = hold(acc + reference(a[:, k0:k0 + KB], b[:, k0:k0 + KB]))
    return acc


# ---- construction ------------------------------------------------------------------------------------------------
def test_mantissa_budget():
    assert [mantissa_bits(k) for k in (64, 256, 1024, 4096, 16384)] == [8, 8, 7, 6, 5]
    assert mantissa_bits(256, extra=2) == 7 and mantissa_bits(64, extra=4) == 7
    with pytest.raises(ValueError):
        exact_operands(128, 256, 1 << 23, 0)


@pytest.mark.parametrize("k", KS)
def test_values_are_bf16_with_p_bits_and_one_exponent_per_row(k):
    p = mantissa_bits(k)
    a, b = _exact(k)
    for x in (a, b):
        x64 = x.double()
        assert x.dtype == torch.bfloat16 and bool((x64 != 0).all())
        assert torch.equal(round_bits(x64, p), x64)                        # at most p significant bits
        assert bool((round_bits(x64, p - 1) != x64).any())                 # and the last of them is used
        e = torch.frexp(x64)[1]
        assert bool((e == e[:, :1]).all())                                 # one exponent per row
        assert int(e.min()) < -8 and int(e.max()) > 8                      # that varies over the rows
        assert float(x64.abs().min()) >= 2.0 ** -12 and float(x64.abs().max()) < 2.0 ** 14
    c = reference(a, b)
    assert torch.equal(c.float().double(), c)                              # the result is an fp32 value


@pytest.mark.parametrize("positive", [False, True], ids=["signed", "positive"])
@pytest.mark.parametrize("k", KS)
def test_exact_under_fp32_accumulation_in_random_orders(k, positive):
    """numpy fp32, one add at a time, in the natural and in three random k orders."""
    a, b = exact_operands(32, 64, k, seed=k, positive=positive)
    want = reference(a, b).numpy()
    prods = (a.float()[:, None, :] * b.float()[None, :, :]).numpy()     # bf16 x bf16: exact in fp32
    rng = np.random.default_rng(k)
    for order in [np.arange(k)] + [rng.permutation(k) for _ in range(3)]:
        acc = np.zeros(prods.shape[:2], dtype=np.float32)
        for i in order:
            acc += prods[:, :, i]
        assert np.array_equal(acc.astype(np.float64), want)


def _tensor_core_adder(a, b, window):
    """fp32 accumulator + 16 products per step: every addend truncated to the ``window``-bit window of the largest
    one, the sum truncated to 24 bits."""
    prods = a.double()[:, None, :] * b.double()[None, :, :]
    acc = torch.zeros(prods.shape[:2], dtype=torch.float64)
    for k0 in range(0, a.shape[1], 16):
        terms = torch.cat([acc[..., None], prods[..., k0:k0 + 16]], -1)
        top = torch.frexp(terms.abs().amax(-1, keepdim=True))[1]
        q = torch.ldexp(torch.ones_like(terms), (top - window).expand_as(terms))
        acc = round_bits(torch.trunc(terms / q).mul(q).sum(-1), 24, "trunc")
    return acc


@pytest.mark.parametrize("k", KS)
def test_exact_under_a_truncating_tensor_core_adder(k):
    a, b = exact_operands(32, 64, k, seed=k + 1)
    want = reference(a, b)
    assert torch.equal(_tensor_core_adder(a, b, 24), want)
    # random signs: the sums stay about sqrt(K) below the worst case the budget allows for, so only a window of about
    # 20 bits or less is seen on this data (21 at K = 256 and 1024, 20 at K = 64 and 4096 for these seeds)
    assert not torch.equal(_tensor_core_adder(a, b, 19), want)
    # all positive: the sums come within a factor of two of the budget, and from K = 256 on (where the budget, not
    # bf16's 8 bits, sets p) every window narrower than 24 bits is seen
    a, b = exact_operands(32, 64, k, seed=k + 1, positive=True)
    want = reference(a, b)
    assert torch.equal(_tensor_core_adder(a, b, 24), want)
    if k >= 256:
        assert not torch.equal(_tensor_core_adder(a, b, 23), want)


def test_rne_bf16_matches_the_fp32_conversion():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1 << 16, generator=g) * torch.exp2(torch.randint(-40, 40, (1 << 16,), generator=g).float())
    ties = (x.view(torch.int32) & ~0xFFFF | 0x8000).view(torch.float32)    # exactly half way between bf16 values
    for v in (x, ties):
        assert torch.equal(rne_bf16(v.double()).view(torch.int16), v.to(torch.bfloat16).view(torch.int16))


def test_bf16_shard_outcomes_match_a_brute_force_loop():
    for world in (1, 2, 3, 4):
        a, b = exact_operands(128, 256, 64 * world, seed=world)
        parts = [reference(a[:2, r * 64:(r + 1) * 64], b[:40, r * 64:(r + 1) * 64]) for r in range(world)]
        got = bf16_shard_outcomes(parts)
        for i, j in itertools.product(range(2), range(40)):
            xs = [torch.tensor(float(c[i, j])).to(torch.bfloat16).float() for c in parts]
            want = set()
            for order in itertools.permutations(range(world)):
                s = torch.tensor(0.0)
                for r in order:
                    s = (s + xs[r]).to(torch.bfloat16).float()             # red.add.bf16: fp32 add, bf16 rounding
                want.add(float(s))
            assert set(got[:, i, j].tolist()) == want


def test_bf16_shard_bound_admits_every_order_and_rejects_a_lost_partial():
    world, k = 8, 64
    a, b = exact_operands(M, N, world * k, seed=9)
    parts = [reference(a[:, r * k:(r + 1) * k], b[:, r * k:(r + 1) * k]) for r in range(world)]
    g = torch.Generator().manual_seed(9)
    for _ in range(20):
        s = torch.zeros_like(parts[0])
        for r in torch.randperm(world, generator=g).tolist():
            s = round_bits(s + round_bits(parts[r], 8), 8)
        assert shard_problems(s, parts) == ""
    assert shard_problems(bf16_shard_outcomes(parts[:4])[0], parts) != ""


# ---- emulated faults: the exact comparison reports them, dyadic data hides some -----------------------------------
def _fault_truncated_bf16(a, b):
    return round_bits(reference(a, b), 8, "trunc"), "bf16"


def _fault_short_operand(a, b):
    return reference(round_bits(a.double(), 4, "trunc"), b), "fp32"


def _fault_bf16_partials(a, b):
    return _blocked(a, b, lambda s: round_bits(s, 8)), "fp32"


def _fault_fp16_partials(a, b):
    return _blocked(a, b, lambda s: round_bits(s, 11)), "fp32"


# fault -> dyadic data hides it at K = 64 / 256 / 1024 / 4096
PRECISION_FAULTS = [(_fault_truncated_bf16, (True, False, False, False)),
                    (_fault_short_operand, (True, True, True, True)),
                    (_fault_bf16_partials, (True, False, False, False)),
                    (_fault_fp16_partials, (True, True, True, True))]


def _reported(fault, a, b):
    got, kind = fault(a, b)
    c = reference(a, b)
    want = rne_bf16(c).double() if kind == "bf16" else c
    return mismatches(got, want) > 0


@pytest.mark.parametrize("fault,hidden", PRECISION_FAULTS, ids=[f.__name__[7:] for f, _ in PRECISION_FAULTS])
def test_precision_fault_is_reported(fault, hidden):
    for k, dyadic_hides in zip(KS, hidden):
        assert _reported(fault, *_exact(k)), f"K = {k}: {fault.__name__} not reported on exact data"
        assert _reported(fault, *dyadic_operands(M, N, k, seed=k)) != dyadic_hides, f"K = {k}, dyadic data"


@pytest.mark.parametrize("num_kb", [5, 6, 7])                  # num_kb mod 4 = 1, 2, 3 of the 4-stage ring
def test_dropped_last_k_block_is_reported(num_kb):
    a, b = _exact(num_kb * KB)
    k = (num_kb - 1) * KB
    assert mismatches(reference(a[:, :k], b[:, :k]), reference(a, b)) > 0


def test_accumulator_not_reset_between_tiles_is_reported():
    a, b = exact_operands(2 * M, N, 256, seed=3)
    c = reference(a, b)
    got = c.clone()
    got[M:] += c[:M]                                   # the CTA's second tile starts from its first tile's sum
    assert mismatches(got, c) > 0


def test_tile_stored_one_epilogue_slice_off_is_reported():
    a, b = _exact(128)
    c = reference(a, b)
    got = c.roll(16, 0)                                # consumer warp ew stores its 16 rows where warp ew+1's go
    assert mismatches(got, c) > 0


@pytest.mark.parametrize("world", [3, 4])
def test_bf16_shard_rounded_once_is_reported(world):
    """A bf16 reduce-scatter that adds the P partials in fp32 and rounds once at the end (at P = 2 that is what the
    two additions into a zeroed shard do anyway).  The ternary operands at K = 64 of the older bf16-shard test keep
    every sum exact in bf16 and cannot tell the two apart."""
    def rounded_once(parts):
        return round_bits(sum(round_bits(c, 8) for c in parts), 8)

    a, b = exact_operands(M, N, 256 * world, seed=world)
    parts = [reference(a[:, r * 256:(r + 1) * 256], b[:, r * 256:(r + 1) * 256]) for r in range(world)]
    assert shard_problems(bf16_shard_outcomes(parts)[-1], parts) == ""
    assert shard_problems(rounded_once(parts), parts) != ""
    g = torch.Generator().manual_seed(world)
    tern = [reference(*(torch.randint(-1, 2, (r, 64), generator=g).to(torch.bfloat16) for r in (M, N)))
            for _ in range(world)]
    assert shard_problems(rounded_once(tern), tern) == ""


def _act32(x, activation):
    """fp32 twin of the epilogue's activation formulas (accurate tanh / exp in place of the approximations)."""
    x = x.float()
    if activation == "gelu":
        return 0.5 * x * (1 + torch.tanh(0.7978845608 * (x + 0.044715 * x * x * x)))
    return x / (1 + torch.exp(-x))


def _activation_data(seed):
    """Rows scaled so that |C| spans about 2^-8 .. 2^8, past silu's overflow point at -87."""
    return exact_operands(M, N, 256, seed, a_exp=(-10, 2), b_exp=(-3, 0))


@pytest.mark.parametrize("activation", ["gelu", "silu"])
def test_activation_after_bf16_rounding_is_reported(activation):
    """bf16 output must be rne_bf16 of the fp32 output of the same launch; an epilogue that rounds C to bf16 before the
    activation fails that, but passes the older flat 2e-2 tolerance on dyadic data."""
    def late(c):
        return rne_bf16(_act32(rne_bf16(c).double(), activation).double())

    c = reference(*_activation_data(5))
    assert float(c.min()) < -87 and float(c.max()) > 87 and float(c.abs().min()) < 2.0 ** -4
    assert mismatches(late(c), rne_bf16(_act32(c, activation).double())) > 0
    cd = reference(*dyadic_operands(512, 512, 128, seed=11))
    assert torch.allclose(late(cd).float(), activation64(cd, activation).float(), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("activation", ["none", "relu", "gelu", "silu"])
def test_activation_bound_accepts_the_documented_error_and_rejects_bf16_inputs(activation):
    c = reference(*_activation_data(6))
    want, bound = activation_bound(c, activation)
    if activation in ("none", "relu"):
        assert bool((bound == 0).all())
        return
    assert bool(((_act32(c, activation).double() - want).abs() <= bound).all())
    # an approximation at the documented limit in the worst direction stays inside
    x = c.float()
    if activation == "gelu":
        arg = 0.7978845608 * (x + 0.044715 * x * x * x)
        t = torch.tanh(arg).double()
        worst = 0.5 * x.double() * (1 + t * (1 - 2.0 ** -10.99 * torch.sign(x.double())))
    else:
        e = torch.exp(-x.double()) * (1 + (2 + torch.floor(1.17 * x.double().abs())) * 2.0 ** -23.1)
        worst = torch.where(x < -87, torch.zeros_like(e), x.double() / (1 + e))
    assert bool(((worst - want).abs() <= bound).all())
    # C rounded to bf16 before the activation is far outside
    late = _act32(rne_bf16(c).double(), activation).double()
    assert int(((late - want).abs() > bound).sum()) > c.numel() // 4


def test_general_bound_admits_fp32_and_truncating_accumulators_but_not_bf16_partials():
    g = torch.Generator().manual_seed(8)
    for k in (512, 4096):
        a = (torch.randn(64, k, generator=g) * torch.exp2(torch.randint(-6, 7, (64, k), generator=g).float()))
        b = (torch.randn(128, k, generator=g) * torch.exp2(torch.randint(-6, 7, (128, k), generator=g).float()))
        a, b = a.to(torch.bfloat16), b.to(torch.bfloat16)
        ref, bound = general_bound(a, b)
        fp32 = (a.float() @ b.float().t()).double()
        trunc = torch.zeros_like(ref)
        for i in range(k):                             # every add truncated to 24 bits
            trunc = round_bits(trunc + a[:, i:i + 1].double() * b[:, i].double(), 24, "trunc")
        assert bool(((fp32 - ref).abs() <= bound).all()) and bool(((trunc - ref).abs() <= bound).all())
        bf16 = _blocked(a, b, lambda s: round_bits(s, 8))
        assert bool(((bf16 - ref).abs() > bound).any())
