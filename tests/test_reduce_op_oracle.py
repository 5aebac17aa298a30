"""tests/reduce_op_oracle.py against brute force, element by element in plain Python: the oracle the op GPU tests
trust must itself be right about IEEE maximum / minimum, signed zeros, canonical NaNs, signed versus unsigned order,
wrapping products, rounded products without flush-to-zero, and each algorithm's order."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests.reduce_op_oracle import (FLOATS, OPS, TYPES, canonical_nan, combine, elem_bytes, kinds, make_inputs,
                                    mismatches, reduce_scatter_expected, ring_expected, rsag_expected, to_bits,
                                    two_shot_expected, values)

_FMT = {"float": (8, 23), "double": (11, 52), "bfloat16": (8, 7), "half": (5, 10)}   # exponent bits, mantissa bits


def _value(bits_, dtype):
    """The exact value of a float's bits as a Fraction (None for NaN, +-inf as float)."""
    e_bits, m_bits = _FMT[dtype]
    sign = -1 if bits_ >> (e_bits + m_bits) else 1
    e = (bits_ >> m_bits) & ((1 << e_bits) - 1)
    m = bits_ & ((1 << m_bits) - 1)
    bias = (1 << (e_bits - 1)) - 1
    if e == (1 << e_bits) - 1:
        return None if m else sign * math.inf
    if e == 0:
        return sign * Fraction(m, 1 << m_bits) * Fraction(2) ** (1 - bias)
    return sign * (1 + Fraction(m, 1 << m_bits)) * Fraction(2) ** (e - bias)


def _round(x, dtype, negative_zero=False):
    """Fraction (or +-inf) rounded to nearest even in the format, as bits: by exhaustive neighbourhood search."""
    e_bits, m_bits = _FMT[dtype]
    bias = (1 << (e_bits - 1)) - 1
    sign_bit = 1 << (e_bits + m_bits)
    if x == math.inf or x == -math.inf:
        return ((e_bits and ((1 << e_bits) - 1)) << m_bits) | (sign_bit if x < 0 else 0)
    if x == 0:
        return sign_bit if negative_zero else 0
    s = sign_bit if x < 0 else 0
    a = abs(x)
    e = max(a.numerator.bit_length() - a.denominator.bit_length(), 1 - bias)   # within one of floor(log2 a)
    while Fraction(2) ** e > a and e > 1 - bias:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    q = Fraction(2) ** (e - m_bits)                 # the spacing of the binade (or of the subnormals)
    k, r = divmod(a, q)
    k = int(k) + (1 if r > q / 2 or (r == q / 2 and int(k) % 2) else 0)
    v = k * q
    if v >= Fraction(2) ** (bias + 1):
        return (((1 << e_bits) - 1) << m_bits) | s
    if v < Fraction(2) ** (1 - bias):
        return s | int(v / Fraction(2) ** (1 - bias - m_bits))
    ee = e + (1 if v >= Fraction(2) ** (e + 1) else 0)
    return s | ((ee + bias) << m_bits) | int((v / Fraction(2) ** ee - 1) * (1 << m_bits))


def _brute(a, b, op, dtype):
    """op on two raw-bit scalars, from the definitions."""
    w = 8 * elem_bytes(dtype)
    if dtype not in FLOATS:
        if op == "prod":
            return (a * b) % (1 << w)
        signed = dtype in ("int", "long", "short")
        x = a - (1 << w) if signed and a >> (w - 1) else a
        y = b - (1 << w) if signed and b >> (w - 1) else b
        return a if (x > y if op == "max" else x < y) else b
    x, y = _value(a, dtype), _value(b, dtype)
    if x is None or y is None:
        return canonical_nan(dtype)
    if op == "prod":
        if (x == 0 and abs(y) == math.inf) or (y == 0 and abs(x) == math.inf):
            return canonical_nan(dtype)
        neg = (a ^ b) >> (w - 1)
        if abs(x) == math.inf or abs(y) == math.inf:
            return _round(-math.inf if neg else math.inf, dtype)
        return _round(x * y, dtype, negative_zero=bool(neg))
    if x == y:                                      # IEEE maximum / minimum order -0 below +0
        return a & b if op == "max" else a | b
    return a if (x > y if op == "max" else x < y) else b


@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("op", OPS)
def test_combine_is_the_definition(op, dtype):
    for kind in kinds(op, dtype):
        va, vb = make_inputs(2, 300, dtype, seed=11, op=op, kind=kind)
        a, b = to_bits(va), to_bits(vb)
        got = combine(a, b, op, dtype)
        for i in range(a.size):
            want = _brute(int(a[i]), int(b[i]), op, dtype)
            assert int(got[i]) == want, (kind, i, hex(int(a[i])), hex(int(b[i])), hex(int(got[i])), hex(want))


def test_signed_zeros_nan_and_signedness():
    f = np.array([0x80000000, 0x00000000, 0x7FC00001, 0xFFC00000], dtype=np.uint32)   # -0, +0, NaN, -NaN
    g = np.array([0x00000000, 0x80000000, 0x3F800000, 0x3F800000], dtype=np.uint32)
    assert combine(f, g, "max", "float").tolist() == [0, 0, 0x7FFFFFFF, 0x7FFFFFFF]
    assert combine(f, g, "min", "float").tolist() == [0x80000000, 0x80000000, 0x7FFFFFFF, 0x7FFFFFFF]
    top = np.array([0x8000], dtype=np.uint16)
    one = np.array([1], dtype=np.uint16)
    assert combine(top, one, "max", "short").tolist() == [1]            # -32768 < 1
    assert combine(top, one, "max", "ushort").tolist() == [0x8000]      # 32768 > 1
    assert combine(np.array([0xFF], np.uint8), np.array([2], np.uint8), "prod", "uchar").tolist() == [0xFE]


def test_products_keep_subnormals():
    x = np.array([np.float32(2.0 ** -63)]).view(np.uint32)
    got = values(combine(x, x, "prod", "float"), "float")[0]
    assert got == np.float32(2.0 ** -126)                                # the smallest normal
    x = np.array([np.float32(2.0 ** -70)]).view(np.uint32)
    y = np.array([np.float32(2.0 ** -60)]).view(np.uint32)
    assert values(combine(x, y, "prod", "float"), "float")[0] == np.float32(2.0 ** -130)   # subnormal, kept


def test_two_shot_16bit_prod_rounds_once():
    """Owner-first fp32 products rounded once differ from a 16-bit rounding per product: the oracle must be the
    former for two-shot and the latter for the rings."""
    world, n = 4, 4096
    vas = make_inputs(world, n, "bfloat16", seed=5, op="prod", kind="near-one")
    ts, rs = two_shot_expected(vas, "prod", "bfloat16"), rsag_expected(vas, "prod", "bfloat16")
    assert mismatches(ts, rs) > 0
    b = [to_bits(v) for v in vas]
    for i in range(0, n, 97):
        s = i * world // n
        acc = np.float32(1.0)
        for q in range(world):
            acc = np.float32(acc * values(b[(s + q) % world][i:i + 1], "bfloat16")[0])
        assert int(to_bits(ts)[i]) == _round(Fraction(float(acc)), "bfloat16", negative_zero=acc < 0)


def test_orders():
    """Ring: rank r folds VA[r], VA[r-1], ...; rsag: segment s folds VA[s+1], ..., VA[s]; two-shot: VA[s], VA[s+1], ...
    -- checked with float products near 1, where the order changes the rounding."""
    world, n = 5, 5 * 64
    vas = make_inputs(world, n, "float", seed=9, op="prod", kind="near-one")
    b = [to_bits(v) for v in vas]

    def fold(order, i):
        acc = values(b[order[0]][i:i + 1], "float")[0]
        for r in order[1:]:
            acc = np.float32(acc * values(b[r][i:i + 1], "float")[0])
        return float(acc)

    for r in range(world):
        got = ring_expected(vas, r, "prod", "float")
        for i in range(0, n, 7):
            assert got[i].item() == fold([(r - t) % world for t in range(world)], i)
    for s in range(world):
        got = reduce_scatter_expected(vas, s, "prod", "float")
        for j in range(0, n // world, 5):
            i = s * n // world + j
            assert got[j].item() == fold([(s + k) % world for k in range(1, world + 1)], i)
    ts = two_shot_expected(vas, "prod", "float")
    for i in range(0, n, 3):
        s = i * world // n
        assert ts[i].item() == fold([(s + q) % world for q in range(world)], i)
    rings = [ring_expected(vas, r, "prod", "float") for r in range(world)]
    assert any(mismatches(rings[0], x) for x in rings[1:])            # the order shows in the bits


def test_inputs_cover_the_hard_cases():
    sp = torch.cat(make_inputs(3, 4000, "half", seed=1, op="max", kind="special")).float()
    assert bool(torch.isnan(sp).any()) and bool(torch.isinf(sp).any())
    assert bool(((sp == 0) & torch.signbit(sp)).any()) and bool(((sp == 0) & ~torch.signbit(sp)).any())
    ex = to_bits(torch.cat(make_inputs(3, 4000, "long", seed=1, op="min", kind="extremes")))
    assert {0x8000000000000000, 0xFFFFFFFFFFFFFFFF} <= set(int(x) for x in ex)
    for dtype in ("float", "bfloat16", "half", "double"):
        vas = make_inputs(2, 4000, dtype, seed=2, op="prod", kind="subnormal")
        p = values(combine(to_bits(vas[0]), to_bits(vas[1]), "prod", dtype), dtype).astype(np.float64)
        tiny = {"float": 2.0 ** -126, "double": 2.0 ** -1022, "bfloat16": 2.0 ** -126, "half": 2.0 ** -14}[dtype]
        assert ((p != 0) & (np.abs(p) < tiny)).sum() > 100, dtype    # subnormal results that an FTZ multiply loses
        vas = make_inputs(2, 4000, dtype, seed=2, op="prod", kind="overflow")
        p = values(combine(to_bits(vas[0]), to_bits(vas[1]), "prod", dtype), dtype)
        assert np.isinf(p).sum() > 100 and (values(to_bits(vas[0]), dtype) == 0).sum() > 10, dtype   # inf * 0 next
