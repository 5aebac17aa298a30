"""tests/loc_oracle.py against brute force on Python values, and its inputs against plausible wrong rules (CPU only)."""
import math
import random

import pytest

from tests.loc_oracle import (LOC_OPS, PAIR_TYPES, KINDS, allreduce_expected, combine, const_expected, const_input,
                              const_vc_init, make_inputs, mismatches, pack, pack_result, unpack, unpack_all)


def _rank_key(op, pair):
    """Brute force: the winner is the max of this key (NaN on top in both ops, -0 below +0, then the smaller index)."""
    v, i = pair
    if isinstance(v, float) and math.isnan(v):
        vk = (1, 0.0, 0)
    else:
        s = 1 if math.copysign(1, v) > 0 else 0
        vk = (0, v if op == "maxloc" else -v, s if op == "maxloc" else 1 - s)
    return vk, -i


def _brute(op, pairs):
    return max(pairs, key=lambda p: _rank_key(op, p))


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
@pytest.mark.parametrize("kind", KINDS)
def test_fold_in_any_order_is_the_brute_force_selection(op, dtype, kind):
    rng = random.Random(7)
    world = 6
    vas = make_inputs(world, 300, dtype, seed=11, kind=kind)
    ranks = [unpack_all(v, dtype) for v in vas]
    want = allreduce_expected(op, vas, dtype)
    brute = b"".join(pack_result(_brute(op, [ranks[r][k] for r in range(world)]), dtype) for k in range(300))
    assert want == brute
    for _ in range(5):   # any combine order and grouping gives the same bits
        order = list(range(world))
        rng.shuffle(order)
        out = []
        for k in range(300):
            items = [ranks[r][k] for r in order]
            while len(items) > 1:
                j = rng.randrange(len(items) - 1)
                items[j:j + 2] = [combine(op, items[j], items[j + 1])]
            out.append(pack_result(items[0], dtype))
        assert b"".join(out) == want


@pytest.mark.parametrize("dtype", PAIR_TYPES)
def test_one_rank_is_a_byte_copy_and_padding_is_zero_after_a_combine(dtype):
    va = make_inputs(1, 50, dtype, seed=3, kind="special")[0]
    assert allreduce_expected("maxloc", [va], dtype) == va
    out = allreduce_expected("maxloc", [va, va], dtype)
    s = len(pack((0, 0), dtype))
    for k in range(0, len(out), s):
        assert out[k:k + s] == pack_result(unpack(out[k:k + s], dtype), dtype)


@pytest.mark.parametrize("dtype", ("float_int", "double_int"))
def test_nan_is_canonical_and_wins_both_ops(dtype):
    nan = float("nan")
    for op in LOC_OPS:
        r = combine(op, (1.0, 5), (-nan, 9))
        assert math.isnan(r[0]) and r[1] == 9
        assert math.isnan(combine(op, (nan, 4), (-nan, 2))[0]) and combine(op, (nan, 4), (-nan, 2))[1] == 2
    b = pack_result((-nan, 3), dtype)
    assert b[:4 if dtype == "float_int" else 8] == (b"\xff\xff\xff\x7f" if dtype == "float_int"
                                                   else b"\xff" * 7 + b"\x7f")


# ------------------------------------------------- wrong rules must show ----
def _wrong(rule):
    def c(op, a, b):
        if rule == "unsigned-index":
            r = combine(op, a, b)
            if (a[0] == b[0] or (isinstance(a[0], float) and math.isnan(a[0]) and math.isnan(b[0]))) and \
                    str(a[0]) == str(b[0]):
                return a if (a[1] & 0xffffffff) <= (b[1] & 0xffffffff) else b
            return r
        if rule in ("first-wins", "last-wins"):
            r = combine(op, a, b)
            tie = str(a[0]) == str(b[0]) or (isinstance(a[0], float) and math.isnan(a[0]) and math.isnan(b[0]))
            return (a if rule == "first-wins" else b) if tie else r
        if rule == "nan-loses":
            na = isinstance(a[0], float) and math.isnan(a[0])
            nb = isinstance(b[0], float) and math.isnan(b[0])
            if na != nb:
                return b if na else a
            return combine(op, a, b)
        if rule == "zeros-equal":
            if a[0] == 0 and b[0] == 0:
                return a if a[1] <= b[1] else b
            return combine(op, a, b)
        raise AssertionError(rule)
    return c


def _fold(c, op, vas, dtype, keep_padding=False):
    ranks = [unpack_all(v, dtype) for v in vas]
    out = []
    for k in range(len(ranks[0])):
        acc, src = ranks[0][k], 0
        for r in range(1, len(ranks)):
            nxt = c(op, acc, ranks[r][k])
            if nxt is ranks[r][k]:
                src = r
            acc = nxt
        if keep_padding:   # "padding copied from an input": the winner's own bytes
            s = len(vas[0]) // len(ranks[0])
            out.append(vas[src][k * s:(k + 1) * s])
        else:
            out.append(pack_result(acc, dtype))
    return b"".join(out)


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_the_inputs_separate_the_oracle_from_wrong_rules(op, dtype):
    rules = ["first-wins", "last-wins", "unsigned-index"]
    if dtype in ("float_int", "double_int"):
        rules += ["nan-loses", "zeros-equal"]
    world = 4
    for rule in rules:
        caught = False
        for kind in KINDS:
            vas = make_inputs(world, 200, dtype, seed=21, kind=kind)
            if mismatches(_fold(_wrong(rule), op, vas, dtype), allreduce_expected(op, vas, dtype), dtype):
                caught = True
        assert caught, rule
    if dtype in ("double_int", "long_int", "short_int"):   # the types with padding bytes
        vas = make_inputs(world, 200, dtype, seed=21, kind="ties")
        assert mismatches(_fold(combine, op, vas, dtype, keep_padding=True), allreduce_expected(op, vas, dtype),
                          dtype)


@pytest.mark.parametrize("op", LOC_OPS)
@pytest.mark.parametrize("world", range(1, 17))
def test_constant_data_check(op, world):
    pairs = [const_input(op, r, world) for r in range(world)]
    acc = pairs[0]
    for p in pairs[1:]:
        acc = combine(op, acc, p)
    assert acc == const_expected(op, world)
    if world >= 2:
        assert combine(op, const_vc_init(op), acc) == const_vc_init(op)           # a kernel that reads VC shows
        by_index = min(pairs, key=lambda p: p[1])
        assert by_index != acc                                                       # index-only selection
    if world >= 3:
        unsigned = min((p for p in pairs if p[0] == acc[0]), key=lambda p: p[1] & 0xffffffff)
        assert unsigned != acc                                                       # unsigned index compare
        last = max((p for p in pairs if p[0] == acc[0]), key=lambda p: p[1])
        assert last != acc                                                           # tie broken the wrong way


def test_pairs_per_layout():
    for dtype, size in zip(PAIR_TYPES, (8, 16, 16, 8, 8)):
        assert len(pack((1, -1), dtype)) == size
    assert pack((-2, 7), "short_int") == b"\xfe\xff\x00\x00\x07\x00\x00\x00"
    assert pack((1.5, -1), "double_int")[8:] == b"\xff\xff\xff\xff\x00\x00\x00\x00"
    assert unpack_all(pack((3, -5), "2int") * 2, "2int") == [(3, -5)] * 2
