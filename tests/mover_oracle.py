"""Exact expected outputs of the data movers: the copy engines (csrc/kernels/p2p.cu), the fused triad + put
(csrc/kernels/fused_triad_put.cu) and the fused command kernel (csrc/kernels/bench_fused.cu).

Every triad body computes ``fmaf(s, c, b)``: ONE rounding of the exact ``b + s*c`` to fp32, round-to-nearest-even,
subnormals kept (the build uses neither ``-ftz`` nor ``--use_fast_math``).  ``fma_f32`` is that value, exactly:

* the fp64 product of two fp32 values is exact (48 significant bits, exponents far inside fp64's range);
* a TwoSum of ``b`` and that product gives ``hi + lo`` == the exact sum;
* ``hi`` rounded to fp32 is the answer unless ``hi`` lies exactly on an fp32 midpoint and ``lo != 0``; then the exact
  sum lies on ``lo``'s side of the midpoint and rounds that way.

Non-finite inputs and results follow plain IEEE arithmetic (inf - inf is NaN, a finite sum beyond the fp32 range is
±inf).

Data sets for the triad (``triad_data``), each index-unique so that a displaced element changes value:

* ``full``: random signs, full 24-bit mantissas, exponents over ±10;
* ``cancel``: ``b = -RN(s*c)``, so ``fma`` returns the rounding error of ``s*c`` where a multiply-then-add returns
  ±0; ``c`` is redrawn where ``s*c`` is exact, so every element tells the two apart (``s`` not a power of two);
* ``special``: ``full`` data with a quarter of the elements replaced by special pairs (``special_pairs``): signed zeros
  whose sign depends on the single rounding, subnormal inputs, subnormal results from normal inputs, finite inputs
  whose result overflows, ±inf inputs, inf - inf, NaN inputs, FLT_MAX, results next to a rounding boundary.

The module also holds the emulated faults the GPU tests must notice (``fault_*``) and the triad payload of
``fill_triad_inputs`` / ``verify_triad`` (``payload_old`` is the periodic one it replaced).
"""
from __future__ import annotations

import numpy as np

F32_MAX = float(np.finfo(np.float32).max)
OVERFLOW_MID = 2.0 ** 128 - 2.0 ** 103          # the fp32 midpoint between FLT_MAX and 2^128
S_VALUES = (3.0, float(np.float32(1.7320508)), -2.375, 2.0 ** -20)   # 3.0 is what every caller passes
# NaN sentinel for float outputs: a quiet NaN with a payload no kernel produces (the GPU's NaN is 0x7fffffff)
SENTINEL_BITS = 0x7FA5C3E1
BYTE_SENTINEL = 0xA5


def f32(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float32)


def bits(x) -> np.ndarray:
    return f32(x).view(np.uint32)


def from_bits(u) -> np.ndarray:
    return np.asarray(u, dtype=np.uint32).view(np.float32)


# ------------------------------------------------------------------------------------------------ fp32 fma ----
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fma_f32(b, c, s) -> np.ndarray:
    """The correctly rounded fp32 value of the exact ``b + s*c`` (= fmaf(s, c, b)), element-wise; ``s`` broadcasts."""
    b, c, s = np.broadcast_arrays(f32(b), f32(c), f32(s))
    with np.errstate(all="ignore"):
        p = s.astype(np.float64) * c.astype(np.float64)
        hi, lo = _two_sum(b.astype(np.float64), p)
        r = hi.astype(np.float32)
        r64 = r.astype(np.float64)
        up = np.nextafter(r, np.float32(np.inf))
        dn = np.nextafter(r, np.float32(-np.inf))
        on_up_mid = hi == (r64 + up.astype(np.float64)) / 2      # hi is the midpoint of (r, up): r < hi
        on_dn_mid = hi == (r64 + dn.astype(np.float64)) / 2      # hi is the midpoint of (dn, r): hi < r
        out = np.where(on_up_mid & (lo > 0), up, np.where(on_dn_mid & (lo < 0), dn, r))
        # the midpoint between ±FLT_MAX and ±2^128 rounds to ±inf, unless the exact sum is a little below it
        edge = (np.abs(hi) == OVERFLOW_MID) & (np.sign(lo) == -np.sign(hi))
        out = np.where(edge, np.copysign(np.float32(F32_MAX), hi).astype(np.float32), out)
    return out.astype(np.float32)


def mul_add_f32(b, c, s) -> np.ndarray:
    """Fault: multiply then add, two roundings (``__fadd_rn(__fmul_rn(s, c), b)``)."""
    b, c, s = np.broadcast_arrays(f32(b), f32(c), f32(s))
    with np.errstate(all="ignore"):
        return (s * c).astype(np.float32) + b


def fma_f32_trunc(b, c, s) -> np.ndarray:
    """Fault: the single rounding truncates (round toward zero) instead of rounding to nearest even."""
    b, c, s = np.broadcast_arrays(f32(b), f32(c), f32(s))
    with np.errstate(all="ignore"):
        p = s.astype(np.float64) * c.astype(np.float64)
        hi, lo = _two_sum(b.astype(np.float64), p)
        r = fma_f32(b, c, s)
        r64 = r.astype(np.float64)
        d = r64 - hi                              # exact: r is within one fp32 ulp of hi
        away = np.where(hi > 0, d > lo, np.where(hi < 0, d < lo, False)) & np.isfinite(r)
        out = np.where(away, np.nextafter(r, np.float32(0)), r)
        overflow = np.isinf(r) & np.isfinite(hi)
        out = np.where(overflow, np.copysign(np.float32(F32_MAX), hi).astype(np.float32), out)
    return out.astype(np.float32)


def _ftz(x):
    x = f32(x)
    tiny = (x != 0) & (np.abs(x) < np.finfo(np.float32).tiny)
    return np.where(tiny, np.copysign(np.float32(0), x), x).astype(np.float32)


def fma_f32_ftz(b, c, s) -> np.ndarray:
    """Fault: subnormal inputs and results flushed to zero (sign kept), as ``-ftz=true`` does."""
    return _ftz(fma_f32(_ftz(b), _ftz(c), s))


# -------------------------------------------------------------------------------------------- data sets ----
def _full(rng, n, spread=10):
    mant = (rng.integers(1 << 23, 1 << 24, n, dtype=np.int64)).astype(np.float64) / (1 << 23)   # [1, 2), 24 bits
    sign = np.where(rng.integers(0, 2, n) == 1, -1.0, 1.0)
    return f32(sign * np.ldexp(mant, rng.integers(-spread, spread + 1, n)))


def special_pairs(s: float):
    """(b, c, what) pairs for one ``s`` whose single rounding is easy to get wrong.  Built for |s| in [2^-20, 4]."""
    s = float(np.float32(s))
    sg = 1.0 if s > 0 else -1.0
    tiny = float(np.float32(2.0 ** -149))
    out = []
    for b in (0.0, -0.0):
        for c in (0.0, -0.0, 1.0, -1.0):
            out.append((b, c, "signed zeros"))
    # s*c below half the smallest subnormal: fma gives ±0 with the sign of s*c, multiply-then-add gives -0 + +0 = +0
    c_small = sg * 2.0 ** -149 / abs(s) / 4
    out += [(0.0, -float(np.float32(c_small)), "zero sign from the single rounding"),
            (-0.0, float(np.float32(c_small)), "zero sign from the single rounding")]
    out += [(tiny, tiny, "subnormal inputs"), (-3 * tiny, 5 * tiny, "subnormal inputs"),
            (float(np.float32(2.0 ** -127)), -1.0, "subnormal input"),
            (1.0, float(np.float32(3 * 2.0 ** -140)), "subnormal c")]
    for k in range(6):   # normal inputs, subnormal result: b + s*RN(-b/s) is the rounding error of -b/s
        b = float(np.float32((1 + k / 7) * 2.0 ** -125))
        out.append((b, float(np.float32(-b / s)), "subnormal result from normal inputs"))
        out.append((-b, float(np.float32(b / s)), "subnormal result from normal inputs"))
    out += [(F32_MAX, sg * F32_MAX, "overflow to +inf"), (-F32_MAX, -sg * F32_MAX, "overflow to -inf"),
            (F32_MAX, -sg * 1.0, "FLT_MAX"), (-F32_MAX, 0.0, "FLT_MAX"), (F32_MAX, -sg * F32_MAX, "FLT_MAX")]
    inf = float("inf")
    out += [(inf, 1.0, "inf input"), (-inf, 2.0, "inf input"), (1.0, inf, "inf input"), (0.5, -inf, "inf input"),
            (inf, sg * -inf, "inf - inf"), (-inf, sg * inf, "inf - inf"), (inf, 0.0, "inf + s*0")]
    nan = float("nan")
    out += [(nan, 1.0, "NaN input"), (1.0, nan, "NaN input"), (nan, nan, "NaN input"), (nan, inf, "NaN input")]
    # exact sums a hair above or below an fp32 midpoint: c = RN(u/2 / s) puts s*c next to half an ulp of b
    for b in (1.0, -1.0, 1.5, float(np.float32(1 + 2.0 ** -23)), 3.0e4, -7.0e-3):
        u = float(np.spacing(np.float32(abs(b))))
        for m in (0.5, 1.5, -0.5):
            out.append((b, float(np.float32(m * u / s)), "next to a rounding boundary"))
    return out


def triad_data(kind: str, n: int, s: float, seed: int = 0):
    """(b, c) float32 arrays of length n for data set ``kind`` and multiplier ``s``."""
    rng = np.random.default_rng([seed, n, {"full": 1, "cancel": 2, "special": 3}[kind]])
    b, c = _full(rng, n), _full(rng, n)
    if kind == "cancel":
        if np.frexp(s)[0] in (0.5, -0.5):
            raise ValueError("cancel data needs an s whose products round (not a power of two)")
        for _ in range(64):     # redraw c where s*c is exact, so every element carries a non-zero rounding error
            with np.errstate(all="ignore"):
                b = -(f32(s) * c).astype(np.float32)
            exact = fma_f32(b, c, s) == 0
            if not exact.any():
                break
            c[exact] = _full(rng, int(exact.sum()))
    elif kind == "special":
        pairs = special_pairs(s)
        where = rng.permutation(n)[: n // 4]
        pick = rng.integers(0, len(pairs), where.size)
        b[where] = f32([pairs[k][0] for k in pick])
        c[where] = f32([pairs[k][1] for k in pick])
    elif kind != "full":
        raise ValueError(kind)
    return b, c


# ---------------------------------------------------------------------------------------- expected outputs ----
def triad_expected(b, c, s, n_put: int | None = None, peer_len: int | None = None, put: bool = True):
    """(local, peer) for triad_put: ``local`` = fma over all of b, c; ``peer`` (length ``peer_len``, default n) holds
    the result over [0, n_put) and the sentinel elsewhere (everywhere without a put)."""
    a = fma_f32(b, c, s)
    n = a.size
    n_put = n if n_put in (None, 0) else n_put
    peer = from_bits(np.full(n if peer_len is None else peer_len, SENTINEL_BITS, dtype=np.uint32)).copy()
    if put:
        peer[:n_put] = a[:n_put]
    return a, peer


def busy_expected(n: int, tripcount: int) -> np.ndarray:
    """The busy command's outputs: its seed ``j`` with tripcount 0 (so out[j] == j shows placement), else the chain's
    closed form (``busy_wait_reference``)."""
    if tripcount == 0:
        return np.arange(n, dtype=np.float32)
    out = np.full(n, np.inf, dtype=np.float32)
    out[0] = 0.0
    return out


# -------------------------------------------------------------------------------------------- the payload ----
def pattern_words(n: int, seed: int) -> np.ndarray:
    """payload.h's pattern_word(i, seed) for i < n, in numpy uint32 arithmetic."""
    i = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = ((i * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)).astype(np.uint32) ^ np.uint32(seed & 0xFFFFFFFF)
        x ^= x >> np.uint32(16)
        x *= np.uint32(0x7FEB352D)
        x ^= x >> np.uint32(15)
        x *= np.uint32(0x846CA68B)
        x ^= x >> np.uint32(16)
    return x


TRIAD_SEED = 0x7A1AD000


def payload(n: int, rank: int):
    """fill_triad_inputs of rank r: b = low 10 bits, c = next 3 bits of pattern word i of seed TRIAD_SEED + r."""
    w = pattern_words(n, TRIAD_SEED + rank)
    return (w & 1023).astype(np.float32), ((w >> 10) & 7).astype(np.float32)


def payload_old(n: int, rank: int):
    """The payload before: b = (i + 17r) & 1023, c = (3i + r) & 7 — both repeat every 1024 elements."""
    i = np.arange(n, dtype=np.int64)
    return ((i + 17 * rank) & 1023).astype(np.float32), ((3 * i + rank) & 7).astype(np.float32)


def verify_triad_count(a, b, c, s: float = 3.0) -> int:
    """verify_triad's rule: a[i] != fmaf(s, c[i], b[i]) (plain float compare)."""
    with np.errstate(invalid="ignore"):
        return int((f32(a) != fma_f32(b, c, s)).sum())


# ------------------------------------------------------------------------------------------ emulated faults ----
def fault_stale_stage(a, tile: int, stages: int):
    """Tile j holds tile j - stages (a stage reused before its new tile arrived)."""
    out = a.copy()
    for j in range(stages, (a.size + tile - 1) // tile):
        lo, hi = j * tile, min((j + 1) * tile, a.size)
        out[lo:hi] = a[lo - stages * tile:hi - stages * tile]
    return out


def fault_displaced_tile(a, tile: int, j: int = 1):
    """Tile j also written at tile j+1's offset (over tile j+1)."""
    out = a.copy()
    lo = (j + 1) * tile
    m = min(tile, a.size - lo)
    out[lo:lo + m] = a[j * tile:j * tile + m]
    return out


def fault_drop_range(a, lo: int, hi: int | None = None, sentinel=None):
    out = a.copy()
    if out.dtype == np.uint8:
        out[lo:hi] = BYTE_SENTINEL if sentinel is None else sentinel
    else:
        out[lo:hi] = from_bits(np.uint32(SENTINEL_BITS)) if sentinel is None else sentinel
    return out


def fault_swap_lanes(a, i: int = 1, j: int = 2):
    """Lanes i and j of every float4 swapped."""
    out = a.copy()
    v = out[: out.size // 4 * 4].reshape(-1, 4)
    v[:, [i, j]] = v[:, [j, i]]
    return out


def fault_interior_put(peer, a, n_put: int, tile: int, which: int = 1):
    """Halo mode: interior tile ``which`` (counted from n_put) also put to the peer at its own offset."""
    out = peer.copy()
    lo = n_put + which * tile
    out[lo:lo + tile] = a[lo:lo + tile]
    return out
