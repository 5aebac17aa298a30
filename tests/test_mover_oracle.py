"""The data movers' oracle (tests/mover_oracle.py) on the CPU: ``fma_f32`` against an exact rational evaluation, the
emulated faults against the expected outputs (each must be seen, with the count the GPU tests would report), and the
triad payload that ``verify_triad`` checks, before and after it stopped repeating every 1024 elements."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import mover_oracle as mo
from tests.field_compare import count_wrong

import torch


def _wrong(got, want) -> int:
    return count_wrong(torch.from_numpy(np.ascontiguousarray(got)), torch.from_numpy(np.ascontiguousarray(want)))


# ------------------------------------------------------------------------------- fma against exact rationals ----
def _round_f32(x: Fraction, zero_sign: float) -> float:
    """Round-to-nearest-even of a rational to fp32, subnormals kept, overflow to ±inf."""
    if x == 0:
        return math.copysign(0.0, zero_sign)
    neg = x < 0
    a = -x if neg else x
    num, den = a.numerator, a.denominator
    e = num.bit_length() - den.bit_length()                  # 2^e <= a < 2^(e+2)
    if (num << max(0, -e)) < (den << max(0, e)):             # a < 2^e
        e -= 1
    q = max(e, -126) - 23                                     # the fp32 quantum at a
    n_, d_ = (num, den << q) if q >= 0 else (num << -q, den)
    m, r = divmod(n_, d_)
    if 2 * r > d_ or (2 * r == d_ and m & 1):
        m += 1
    v = math.ldexp(m, q) if m.bit_length() + q <= 1024 else math.inf
    if v >= 2.0 ** 128:
        v = math.inf
    return -v if neg else v


def _exact_fma(b: float, c: float, s: float) -> float:
    if not (math.isfinite(b) and math.isfinite(c) and math.isfinite(s)):
        return float(np.float32(np.float64(b) + np.float64(s) * np.float64(c)))   # IEEE on inf / NaN
    p_neg = math.copysign(1.0, s) * math.copysign(1.0, c) < 0
    both_neg_zero = b == 0 and math.copysign(1.0, b) < 0 and s * c == 0 and p_neg
    return _round_f32(Fraction(b) + Fraction(s) * Fraction(c), -1.0 if both_neg_zero else 1.0)


def _check_exact(b, c, s):
    b, c = mo.f32(b), mo.f32(c)
    got = mo.fma_f32(b, c, s)
    s_arr = np.broadcast_to(mo.f32(s), b.shape)
    want = mo.f32([_exact_fma(float(x), float(y), float(z)) for x, y, z in zip(b, c, s_arr)])
    bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want)))
    assert bad.size == 0, [(float(b[i]), float(c[i]), float(s_arr[i]), float(got[i]), float(want[i]))
                           for i in bad[:5]]


N_EXACT = 100_000


@pytest.mark.parametrize("kind", ["full", "cancel", "special"])
def test_fma_f32_equals_exact_rational_on_each_data_set(kind):
    per = N_EXACT // 3 + 1
    for k, s in enumerate(mo.S_VALUES[:3]):
        b, c = mo.triad_data(kind, per, s, seed=k)
        _check_exact(b, c, s)


def test_fma_f32_equals_exact_rational_on_random_bit_patterns():
    """Any fp32 bit patterns: subnormals, overflow, inf and NaN included, s drawn the same way."""
    rng = np.random.default_rng(11)
    n = N_EXACT
    b = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    c = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    s = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    _check_exact(b, c, s)
    # the same near the subnormal range and near the top of the range, where the random draw is thin
    e = rng.integers(-160, -100, n)
    b = mo.f32(np.ldexp(rng.uniform(-2, 2, n), e))
    c = mo.f32(np.ldexp(rng.uniform(-2, 2, n), rng.integers(-30, 0, n)))
    _check_exact(b, c, mo.f32(np.ldexp(rng.uniform(-2, 2, n), rng.integers(-60, -20, n))))
    b = mo.f32(np.ldexp(rng.uniform(-2, 2, n), rng.integers(120, 128, n)))
    _check_exact(b, c, mo.f32(np.ldexp(rng.uniform(-2, 2, n), rng.integers(100, 150, n) - 30)))


def test_fma_f32_hand_picked_midpoints():
    """Exact sums on an fp32 midpoint (ties to even) and a hair off one (rounds toward the hair), in the normal and
    the subnormal range and at the overflow threshold; the fp64 sum alone rounds half of these the wrong way."""
    u = 2.0 ** -23
    cases = [
        (1.0, 2.0 ** -24, 1.0, 1.0),                               # tie -> even (down)
        (1.0 + u, 2.0 ** -24, 1.0, 1.0 + 2 * u),                   # tie -> even (up)
        (2.0 ** 30 + 2.0 ** 7, 1 - u, 2.0 ** 6 * (1 + u), 2.0 ** 30 + 2.0 ** 7),   # hair below the tie
        (2.0 ** 30 + 3 * 2.0 ** 7, -(1 - u), 2.0 ** 6 * (1 + u), 2.0 ** 30 + 3 * 2.0 ** 7),   # hair above
        (-(2.0 ** 30 + 2.0 ** 7), -(1 - u), 2.0 ** 6 * (1 + u), -(2.0 ** 30 + 2.0 ** 7)),
        (2.0 ** -140 + 2.0 ** -149, 2.0 ** -120 * (1 - u), 2.0 ** -30 * (1 + u), 2.0 ** -140 + 2.0 ** -149),
        (2.0 ** -140 + 2.0 ** -149, 2.0 ** -120, 2.0 ** -30, 2.0 ** -140 + 2.0 ** -148),   # subnormal tie -> even
        (mo.F32_MAX, 1.0, 2.0 ** 103, math.inf),                   # the overflow midpoint: ties to 2^128 -> inf
        (mo.F32_MAX, 1 - u, 2.0 ** 103 * (1 + u), mo.F32_MAX),     # a hair below it stays finite
        (0.0, -(2.0 ** -149), 0.25, -0.0),                         # underflow keeps the sign of s*c
    ]
    for b, c, s, want in cases:
        assert float(np.float32(s)) == s and float(np.float32(c)) == c and float(np.float32(b)) == b
        got = float(mo.fma_f32(b, c, s))
        assert got == want and math.copysign(1, got) == math.copysign(1, want), (b, c, s, got, want)
        assert _exact_fma(b, c, s) == want
    naive = [float(np.float32(np.float64(b) + np.float64(s) * np.float64(c))) for b, c, s, _ in cases]
    assert sum(x != w for x, (_, _, _, w) in zip(naive, cases)) >= 3


def test_special_pairs_cover_every_class():
    for s in mo.S_VALUES:
        pairs = mo.special_pairs(s)
        b, c = mo.f32([p[0] for p in pairs]), mo.f32([p[1] for p in pairs])
        a = mo.fma_f32(b, c, s)
        whats = {p[2] for p in pairs}
        assert {"signed zeros", "subnormal inputs", "subnormal result from normal inputs", "overflow to +inf",
                "inf - inf", "NaN input", "FLT_MAX", "next to a rounding boundary"} <= whats
        assert np.isnan(a).sum() >= 6 and np.isposinf(a).any() and np.isneginf(a).any()
        assert (np.signbit(a) & (a == 0)).any() and (~np.signbit(a) & (a == 0)).any()
        sub = (a != 0) & (np.abs(a) < np.finfo(np.float32).tiny)
        assert sub.sum() >= (2 if abs(np.frexp(s)[0]) == 0.5 else 6), s
        _check_exact(b, c, s)


# ------------------------------------------------------------------------------------------ emulated faults ----
N = 3 * 4096 + 3 * 1024 + 7


@pytest.mark.parametrize("s", mo.S_VALUES[:3])
def test_multiply_then_add_is_seen(s):
    b, c = mo.triad_data("cancel", N, s)
    want = mo.fma_f32(b, c, s)
    fault = mo.mul_add_f32(b, c, s)
    assert (fault == 0).all()                               # two roundings cancel exactly ...
    assert _wrong(fault, want) == N and (want != 0).all()   # ... the single one leaves the error
    for kind in ("full", "special"):
        b, c = mo.triad_data(kind, N, s)
        assert _wrong(mo.mul_add_f32(b, c, s), mo.fma_f32(b, c, s)) >= 0.02 * N, kind
    b, c = mo.triad_data("special", N, s)
    assert _wrong(mo.mul_add_f32(b, c, s), mo.fma_f32(b, c, s)) > 0


@pytest.mark.parametrize("kind", ["full", "special"])
def test_truncation_is_seen(kind):
    """(Not on ``cancel``: there the result is an exact rounding error, which no rounding mode changes.)"""
    s = 3.0
    b, c = mo.triad_data(kind, N, s)
    want = mo.fma_f32(b, c, s)
    fault = mo.fma_f32_trunc(b, c, s)
    differ = _wrong(fault, want)
    assert differ >= 0.2 * N, differ              # about half the inexact results round away from zero
    fin = np.isfinite(want)
    assert (np.abs(fault[fin]) <= np.abs(want[fin])).all()


def test_ftz_is_seen_only_on_special_data():
    for s in mo.S_VALUES[:3]:
        b, c = mo.triad_data("special", N, s)
        want = mo.fma_f32(b, c, s)
        fault = mo.fma_f32_ftz(b, c, s)
        sub = np.isfinite(want) & (want != 0) & (np.abs(want) < np.finfo(np.float32).tiny)
        assert _wrong(fault, want) >= int(sub.sum()) > 20
        b, c = mo.triad_data("full", N, s)
        assert _wrong(mo.fma_f32_ftz(b, c, s), mo.fma_f32(b, c, s)) == 0


@pytest.mark.parametrize("kind", ["full", "cancel", "special"])
def test_placement_faults_are_seen(kind):
    s = 3.0
    b, c = mo.triad_data(kind, N, s)
    a = mo.fma_f32(b, c, s)
    tile = 1024                                               # a 4 KiB stage
    stale = mo.fault_stale_stage(a, tile, 2)
    moved = N - 2 * tile
    # cancel's values are rounding errors of a few significant bits, so some displaced ones happen to be equal
    seen = {"full": 0.99, "cancel": 0.9, "special": 0.7}[kind]
    assert _wrong(stale, a) >= seen * moved
    assert _wrong(mo.fault_displaced_tile(a, tile), a) >= seen * tile
    last = N // tile * tile
    assert _wrong(mo.fault_drop_range(a, last), a) == N - last           # the last partial tile dropped
    assert _wrong(mo.fault_drop_range(a, N & ~3), a) == N % 4 == 3        # the fused triad's n % 4 tail
    swapped = mo.fault_swap_lanes(a)
    assert _wrong(swapped, a) == 2 * _wrong(a[1:N & ~3:4], a[2:N & ~3:4])
    assert _wrong(swapped, a) >= 0.6 * (N // 2)


def test_copy_tail_and_interior_put_are_seen():
    rng = np.random.default_rng(5)
    for nbytes in (17, 31, 4096 + 15, 65536 + 12):
        src = rng.integers(0, 256, nbytes, dtype=np.uint8)
        src[src == mo.BYTE_SENTINEL] = 0
        dropped = mo.fault_drop_range(src, nbytes & ~15)
        assert int((dropped != src).sum()) == nbytes % 16
    n_put, tile = 4 * 4096, 4096
    b, c = mo.triad_data("full", 3 * n_put, 3.0)
    a, peer = mo.triad_expected(b, c, 3.0, n_put=n_put, peer_len=3 * n_put)
    assert _wrong(peer[:n_put], a[:n_put]) == 0
    assert (peer[n_put:].view(np.uint32) == mo.SENTINEL_BITS).all()
    fault = mo.fault_interior_put(peer, a, n_put, tile)
    assert int((fault.view(np.uint32) != peer.view(np.uint32)).sum()) == tile
    _, none = mo.triad_expected(b, c, 3.0, put=False)
    assert (none.view(np.uint32) == mo.SENTINEL_BITS).all()


def test_sentinel_is_a_nan_no_fma_returns():
    x = mo.from_bits(np.uint32(mo.SENTINEL_BITS))
    assert np.isnan(x) and mo.SENTINEL_BITS != 0x7FFFFFFF and mo.SENTINEL_BITS != 0x7FC00000


def test_busy_expected_is_the_package_reference():
    from hpc_patterns_b200.ops.payload import busy_wait_reference

    for trip in (0, 1, 2):
        assert np.array_equal(mo.busy_expected(300, trip), busy_wait_reference(300, trip).numpy())


# ------------------------------------------------------------------------------------------------ the payload ----
NP = (1 << 21) + 4096 + 7


def _moves(n):
    """name -> (shift in elements, faulty-index range): 4, 16 and 64 KiB blocks moved by their own size, and a stale
    stage of the default TMA ring (6 stages of 16 KiB)."""
    return {"4 KiB block": (1024, range(8192, 8192 + 1024)), "16 KiB block": (4096, range(16384, 16384 + 4096)),
            "64 KiB block": (16384, range(65536, 65536 + 16384)),
            "stale stage": (6 * 4096, range(6 * 4096 * 3, 6 * 4096 * 3 + 4096))}


def _apply_move(a, shift, where):
    out = a.copy()
    idx = np.asarray(where)
    out[idx] = a[idx - shift]
    return out


def test_old_payload_hides_displacement():
    for rank in (0, 5):
        b, c = mo.payload_old(NP, rank)
        a = mo.fma_f32(b, c, 3.0)
        assert mo.verify_triad_count(a, b, c) == 0
        for name, (shift, where) in _moves(NP).items():
            assert mo.verify_triad_count(_apply_move(a, shift, where), b, c) == 0, name
        assert mo.verify_triad_count(mo.fault_stale_stage(a, 4096, 6), b, c) == 0


def test_new_payload_reports_displacement_exactly():
    for rank in (0, 5):
        b, c = mo.payload(NP, rank)
        a = mo.fma_f32(b, c, 3.0)
        assert mo.verify_triad_count(a, b, c) == 0
        for name, (shift, where) in _moves(NP).items():
            moved = _apply_move(a, shift, where)
            count = mo.verify_triad_count(moved, b, c)
            assert count == int((moved != a).sum()) >= 0.99 * len(where), name
        stale = mo.fault_stale_stage(a, 4096, 6)
        assert mo.verify_triad_count(stale, b, c) >= 0.99 * (NP - 6 * 4096)


def test_new_payload_has_no_short_period_small_integers_and_differs_per_rank():
    b, c = mo.payload(NP, 0)
    a = b + 3 * c
    assert np.array_equal(a, mo.fma_f32(b, c, 3.0))               # b + 3c is exact
    assert (b == np.floor(b)).all() and (c == np.floor(c)).all()
    assert b.min() == 0 and b.max() == 1023 and c.min() == 0 and c.max() == 7
    for k in range(21):
        sh = 1 << k
        assert (a[sh:] != a[:-sh]).mean() >= 0.99, sh
    ranks = [mo.fma_f32(*mo.payload(1 << 16, r), 3.0) for r in range(8)]
    for r in range(8):
        for q in range(r):
            assert (ranks[r] != ranks[q]).mean() >= 0.99, (r, q)


def test_payload_twins_agree():
    """The package's twin (built on pattern_reference) and this numpy one, and the hash itself."""
    from hpc_patterns_b200.ops.fused import TRIAD_SEED, triad_inputs_reference
    from hpc_patterns_b200.ops.p2p import pattern_reference

    assert TRIAD_SEED == mo.TRIAD_SEED
    assert np.array_equal(pattern_reference(4099, 0xDEADBEEF).numpy().astype(np.uint32),
                          mo.pattern_words(4099, 0xDEADBEEF))
    for rank in (0, 1, 5):
        tb, tc = triad_inputs_reference(10007, rank)
        b, c = mo.payload(10007, rank)
        assert np.array_equal(tb.numpy(), b) and np.array_equal(tc.numpy(), c)
