"""The rules of maxloc / minloc (↔ MPI_MAXLOC / MPI_MINLOC) on the value-index pair types, as code.

A pair is (value, index) in the C struct of its type, natural layout, padding bytes zero in every combined pair:

    type        value    size  index at   pairs per 16-byte vector
    float_int   float    8     4          2
    double_int  double   16    8          1
    long_int    int64    16    8          1
    2int        int32    8     4          2
    short_int   int16    8     4          2      (bytes 2-3 are padding)

(u,i) o (v,j): the larger (maxloc) or smaller (minloc) value wins; floats in max / min's order (-0 < +0), a NaN value
wins in both and every NaN ties with every NaN; equal values (bit-equal, or both NaN) take the smaller signed index.
The result's NaN is the canonical one (all bits set but the sign).  That makes the combine a selection under a total
order, so every algorithm and combine order gives the same bits: at P >= 2 every element is that selection, packed;
at P = 1 VC is a byte copy of VA (padding and NaN payloads untouched).
"""
import math
import random
import struct

import numpy as np

PAIR_TYPES = ("float_int", "double_int", "long_int", "2int", "short_int")
LOC_OPS = ("maxloc", "minloc")
# type -> (struct format of the value, bytes per pair, offset of the index, floating?)
LAYOUT = {"float_int": ("<f", 8, 4, True), "double_int": ("<d", 16, 8, True), "long_int": ("<q", 16, 8, False),
          "2int": ("<i", 8, 4, False), "short_int": ("<h", 8, 4, False)}
VALUE_BITS = {"float_int": 32, "double_int": 64, "long_int": 64, "2int": 32, "short_int": 16}
CANONICAL_NAN = {"float_int": b"\xff\xff\xff\x7f", "double_int": b"\xff\xff\xff\xff\xff\xff\xff\x7f"}
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


def pair_bytes(dtype):
    return LAYOUT[dtype][1]


def pairs_per_vector(dtype):
    return 16 // pair_bytes(dtype)


# ---------------------------------------------------------------- layout ----
def pack(pair, dtype, pad=b""):
    """The bytes of one pair; ``pad`` fills the padding bytes (zero by default)."""
    fmt, size, off, fl = LAYOUT[dtype]
    v, i = pair
    vb = struct.pack(fmt, v)
    buf = bytearray(size)
    buf[:len(vb)] = vb
    buf[off:off + 4] = struct.pack("<i", i)
    holes = [k for k in range(size) if not (k < len(vb) or off <= k < off + 4)]
    for k, b in zip(holes, pad):
        buf[k] = b
    return bytes(buf)


def unpack(b, dtype):
    fmt, size, off, _ = LAYOUT[dtype]
    return struct.unpack(fmt, b[:struct.calcsize(fmt)])[0], struct.unpack("<i", b[off:off + 4])[0]


def value_of_bits(bits, dtype):
    """A value given by its raw bits (for NaN payloads and signed zeros)."""
    fmt = LAYOUT[dtype][0]
    n = struct.calcsize(fmt)
    return struct.unpack(fmt, bits.to_bytes(n, "little"))[0]


def pack_all(pairs, dtype, pads=None):
    return b"".join(pack(p, dtype, pads[k] if pads else b"") for k, p in enumerate(pairs))


def unpack_all(buf, dtype):
    s = pair_bytes(dtype)
    return [unpack(buf[k:k + s], dtype) for k in range(0, len(buf), s)]


# --------------------------------------------------------------- combine ----
def _is_nan(v):
    return isinstance(v, float) and math.isnan(v)


def value_cmp(u, v):
    """-1, 0, 1: u against v in the value order (-0 < +0; NaN above everything, all NaNs equal)."""
    nu, nv = _is_nan(u), _is_nan(v)
    if nu or nv:
        return 0 if nu and nv else (1 if nu else -1)
    if u == v:
        if isinstance(u, float) and math.copysign(1, u) != math.copysign(1, v):
            return 1 if math.copysign(1, u) > 0 else -1
        return 0
    return 1 if u > v else -1


def combine(op, a, b):
    """(u,i) o (v,j) on Python values; the result's value is canonical (NaN stays NaN: packing makes it canonical)."""
    c = value_cmp(a[0], b[0])
    if op == "minloc" and not (_is_nan(a[0]) or _is_nan(b[0])):
        c = -c            # NaN still wins
    if c > 0:
        return a
    if c < 0:
        return b
    return a if a[1] <= b[1] else b


def pack_result(pair, dtype):
    """A combined pair's bytes: padding zero, a NaN value canonical."""
    if _is_nan(pair[0]):
        b = bytearray(pack((0.0, pair[1]), dtype))
        nb = CANONICAL_NAN[dtype]
        b[:len(nb)] = nb
        return bytes(b)
    return pack(pair, dtype)


def allreduce_expected(op, vas, dtype):
    """VC bytes of every rank after an allreduce of ``vas`` (the bytes of each rank's VA), whatever the algorithm."""
    if len(vas) == 1:
        return bytes(vas[0])
    ranks = [unpack_all(v, dtype) for v in vas]
    out = []
    for k in range(len(ranks[0])):
        acc = ranks[0][k]
        for r in range(1, len(ranks)):
            acc = combine(op, acc, ranks[r][k])
        out.append(pack_result(acc, dtype))
    return b"".join(out)


def combine_expected(op, vc, va, dtype):
    """VC = op(VC, VA) element by element (the unfused ring's combine, and ``accumulate``)."""
    a, b = unpack_all(vc, dtype), unpack_all(va, dtype)
    return b"".join(pack_result(combine(op, x, y), dtype) for x, y in zip(a, b))


def mismatches(got, want, dtype):
    """Pairs whose bytes differ."""
    s = pair_bytes(dtype)
    g = np.frombuffer(bytes(got), np.uint8).reshape(-1, s)
    w = np.frombuffer(bytes(want), np.uint8).reshape(-1, s)
    return int((g != w).any(axis=1).sum())


def describe(got, want, dtype, limit=4):
    s = pair_bytes(dtype)
    bad = [k for k in range(len(want) // s) if got[k * s:(k + 1) * s] != want[k * s:(k + 1) * s]]
    return f"{len(bad)} pairs differ, first: " + ", ".join(
        f"#{k}: got {got[k * s:(k + 1) * s].hex()} want {want[k * s:(k + 1) * s].hex()}" for k in bad[:limit])


# ---------------------------------------------------------------- inputs ----
KINDS = ("ties", "special", "zeros", "wide")


def _value(dtype, kind, rng):
    fl = LAYOUT[dtype][3]
    bits = VALUE_BITS[dtype]
    lo, hi = -2 ** (bits - 1), 2 ** (bits - 1) - 1
    if kind == "ties":                      # a tiny set: most elements tie with another rank's
        return float(rng.choice((-1.0, 0.0, 2.0))) if fl else rng.choice((-1, 0, 2))
    if kind == "zeros":                     # signed zeros next to the values just above and below them
        return rng.choice((0.0, -0.0, 1.0, -1.0)) if fl else rng.choice((0, -1, 1))
    if kind == "special":
        if fl:
            nans = [value_of_bits(b, dtype) for b in ((0x7fc00001, 0xffc00000, 0x7f800001) if bits == 32 else
                                                      (0x7ff8000000000001, 0xfff8000000000000, 0x7ff0000000000001))]
            return rng.choice([0.0, -0.0, math.inf, -math.inf, 1.0, -1.0] + nans)
        return rng.choice((lo, hi, 0, -1, 1))
    return rng.uniform(-1e3, 1e3) if fl else rng.randint(lo, hi)


def _index(kind, rng):
    if kind == "wide":
        return rng.randint(INT_MIN, INT_MAX)
    return rng.choice((INT_MIN, INT_MAX, -1, 0, 1, -2, 3))


def make_inputs(world, n, dtype, seed, kind, garbage_padding=True):
    """VA bytes of every rank: n pairs of the given kind; the padding bytes hold garbage unless told otherwise."""
    rng = random.Random(seed)
    holes = pair_bytes(dtype) - struct.calcsize(LAYOUT[dtype][0]) - 4
    out = []
    for _ in range(world):
        pairs = [(_value(dtype, kind, rng), _index(kind, rng)) for _ in range(n)]
        pads = [bytes(rng.randrange(256) for _ in range(holes)) if garbage_padding else b"" for _ in range(n)]
        out.append(pack_all(pairs, dtype, pads))
    return out


# ------------------------------------------------------ constant-data check ----
def const_input(op, rank, world):
    """(value, index) rank holds in the miniapps' constant-data run."""
    mx = op == "maxloc"
    return ((0 if mx else 1), -world - 10) if rank == 0 else ((1 if mx else 0), 2 * rank - 3)


def const_expected(op, world):
    return const_input(op, 0, 1) if world == 1 else ((1 if op == "maxloc" else 0), -1)


def const_vc_init(op):
    return (7 if op == "maxloc" else -7), -1000
