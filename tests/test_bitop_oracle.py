"""tests/bitop_oracle.py against brute force on Python ints, its inputs against the faults they must expose, and the
miniapps' constant-data check of band / bor / bxor / land / lor / lxor."""
import numpy as np
import pytest
import torch

from hpc_patterns_b200.models import allreduce as ar
from tests.bitop_oracle import (BIT_OPS, CHECK_VC, INT_TYPES, KINDS, LOGICAL_OPS, allreduce_expected, brute_force,
                                check_expected, check_input, combine, combine_expected, make_inputs, mismatches,
                                reduce_scatter_expected)
from tests.reduce_op_oracle import elem_bytes, to_bits
from tests.rsag_oracle import segment


def _ints(t):
    return [int(x) for x in to_bits(t)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_oracle_matches_brute_force(op, dtype, kind):
    for world in (1, 2, 3, 5, 8):
        vas = make_inputs(world, 96, dtype, seed=world, kind=kind)
        got = _ints(allreduce_expected(vas, op, dtype))
        assert got == brute_force([_ints(v) for v in vas], op, dtype), (world, op, dtype, kind)


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_one_rank_is_va(op, dtype):
    """One rank: VC is a copy of VA, unnormalised even for the logical ops."""
    va = make_inputs(1, 64, dtype, seed=9, kind="dense")
    assert mismatches(allreduce_expected(va, op, dtype), va[0]) == 0


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_every_order_gives_the_same_bits(op, dtype):
    """The op is commutative and associative: any rotation or reversal of the ranks folds to the same result."""
    vas = make_inputs(5, 200, dtype, seed=4, kind="sparse")
    want = allreduce_expected(vas, op, dtype)
    for order in ([2, 3, 4, 0, 1], [4, 3, 2, 1, 0], [1, 0, 3, 2, 4]):
        assert mismatches(allreduce_expected([vas[i] for i in order], op, dtype), want) == 0
    for s in range(5):
        seg = segment(200, 5, s)
        assert mismatches(reduce_scatter_expected(vas, s, op, dtype), want[seg]) == 0


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_combine_expected(op, dtype):
    vc, va = make_inputs(2, 77, dtype, seed=5, kind="high")
    assert _ints(combine_expected(vc, va, op, dtype)) == brute_force([_ints(vc), _ints(va)], op, dtype)


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", LOGICAL_OPS)
def test_logical_results_take_both_values(op, dtype):
    """Zero-heavy inputs: at every rank count, every logical result is 0 somewhere and 1 somewhere."""
    for kind in ("sparse", "high"):
        for world in range(2, 9):
            r = to_bits(allreduce_expected(make_inputs(world, 512, dtype, seed=world, kind=kind), op, dtype))
            assert set(np.unique(r).tolist()) == {0, 1}, (kind, world)


def _wrong_truths(nb):
    """Truth tests that look at less or more than one element: one part of it (a byte, or a 32-bit half of a 64-bit
    lane), or the whole 32-bit word around a narrow element."""
    out = {}
    for part in (1, 4) if nb == 8 else (1,) if nb > 1 else ():
        per = nb // part
        for which in range(per):
            out[f"part{part}[{which}]"] = (lambda b, part=part, per=per, which=which:
                                           b.view({1: np.uint8, 4: np.uint32}[part]).reshape(-1, per)[:, which] != 0)
    if nb < 4:
        out["word"] = lambda b: np.repeat(b.view(np.uint32) != 0, 4 // nb)
    return out


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", LOGICAL_OPS)
def test_inputs_catch_partial_truth(op, dtype):
    """Zero-heavy data with high-part-only values next to zeros: a logical op that tests truth per byte, per 32-bit
    word or per 32-bit half instead of per element disagrees with the oracle."""
    nb = elem_bytes(dtype)
    world, n = 4, 4096
    vas = [torch.cat([h, s]) for h, s in zip(make_inputs(world, n, dtype, seed=11, kind="high"),
                                             make_inputs(world, n, dtype, seed=12, kind="sparse"))]
    bits = [to_bits(v) for v in vas]
    want = to_bits(allreduce_expected(vas, op, dtype)).astype(bool)
    for name, truth in _wrong_truths(nb).items():
        acc = truth(bits[0])
        for b in bits[1:]:
            acc = {"land": acc & truth(b), "lor": acc | truth(b), "lxor": acc ^ truth(b)}[op]
        assert (acc != want).any(), name


@pytest.mark.parametrize("dtype", INT_TYPES)
def test_high_kind_is_high_part_only(dtype):
    nb = elem_bytes(dtype)
    b = np.concatenate([to_bits(v) for v in make_inputs(3, 2048, dtype, seed=2, kind="high")]).astype(np.uint64)
    nz = b[b != 0]
    assert (b == 0).any() and nz.size
    low_mask = np.uint64((1 << (8 * nb - 8)) - 1)
    if nb == 8:
        assert ((nz & np.uint64(0xFFFFFFFF)) == 0).all()     # top 32 bits only ...
        assert ((nz & low_mask) == 0).any() and ((nz & low_mask) != 0).any()   # ... top byte only among them
    elif nb > 1:
        assert ((nz & low_mask) == 0).all()


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_combine_is_lane_local(op, dtype):
    """One lane's result depends on that lane's inputs only (no carries or borrows between lanes)."""
    a, b = make_inputs(2, 64, dtype, seed=8, kind="dense")
    ab, bb = to_bits(a), to_bits(b)
    full = combine(ab, bb, op, dtype)
    for i in (0, 17, 63):
        assert combine(ab[i:i + 1], bb[i:i + 1], op, dtype)[0] == full[i]


# ------------------------------------------------------ constant-data check ----
@pytest.mark.parametrize("op", BIT_OPS)
def test_constant_check(op):
    """Exact in uchar for 1..16 ranks; the Python twin agrees; VC before the run is not the result."""
    for world in range(1, 17):
        vals = [check_input(op, r) for r in range(world)]
        assert all(0 <= v <= 255 for v in vals)
        want = check_expected(op, world)
        assert brute_force([[v] for v in vals], op, "uchar") == [want]
        assert ar.expected_value(world, op) == want
        assert [ar.op_input(op, r, world) for r in range(world)] == vals
        assert ar.vc_init(op, world) == CHECK_VC[op] != want


@pytest.mark.parametrize("bitwise,logical", [("band", "land"), ("bor", "lor"), ("bxor", "lxor")])
def test_constant_check_tells_bitwise_from_logical(bitwise, logical):
    for world in range(2, 17):
        for op, other in ((bitwise, logical), (logical, bitwise)):
            vals = [[check_input(op, r)] for r in range(world)]
            assert brute_force(vals, other, "uchar") != [check_expected(op, world)], (op, world)


def test_refusals():
    for dtype in ("float", "double", "bfloat16", "half"):
        with pytest.raises(ValueError, match="integer types only"):
            make_inputs(2, 8, dtype, seed=0, kind="dense")
    with pytest.raises(ValueError, match="unknown op"):
        combine(np.zeros(2, np.uint32), np.zeros(2, np.uint32), "avg", "int")
