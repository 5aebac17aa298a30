"""Fields and planted faults for the halo checks, shared by the GPU tests (tests/test_gpu_verifiers.py) and their CPU
twins on the emulated device (tests/test_verifier_rule.py).

``value_row`` is a row whose reference step, at ``alpha = s = 1`` with both neighbour rows all -0, is the row itself
(``x*1 + (-0 + -0) = x`` for every x, -0 and NaN included), so a one-row slab plants any wanted value exactly.
``special_step`` is a slab drawn from a palette of ±0, subnormals, the largest finite values, ±inf and NaN, whose
reference step produces all of those.  ``GROW`` / ``DECAY`` are the runs of the closed-form field into inf and NaN and
through subnormals into ±0, with their checkpoints.
"""
import numpy as np
import torch

from hpc_patterns_b200.models.halo import initial_field, reference_steps

TYPES = (torch.float32, torch.float64, torch.bfloat16, torch.float16)
_INT = {2: torch.int16, 4: torch.int32, 8: torch.int64}
_NP_U = {2: np.uint16, 4: np.uint32, 8: np.uint64}
_NP_I = {2: np.int16, 4: np.int32, 8: np.int64}
_INF = {torch.float32: 0x7F800000, torch.float64: 0x7FF0000000000000, torch.bfloat16: 0x7F80, torch.float16: 0x7C00}
_QUIET = {torch.float32: 0x00400000, torch.float64: 0x0008000000000000, torch.bfloat16: 0x0040, torch.float16: 0x0200}

# (alpha, s, checkpoints): the growing run reaches inf and NaN (fp64 needs a faster growth to get there), the decaying
# run has subnormals at the first checkpoint and only ±0 at the second.  The slab geometries of the tests (26 or 27
# global rows) are the ones these were chosen for; the tests assert that the values are there.
GROW = {torch.float16: (0.3, 0.7, (22, 40)), torch.bfloat16: (0.3, 0.7, (176, 200)),
        torch.float32: (0.3, 0.7, (176, 200)), torch.float64: (3.0, 7.0, (256, 300))}
DECAY = {torch.float16: (0.1, 0.1, (13, 20)), torch.bfloat16: (0.1, 0.1, (76, 100)),
         torch.float32: (0.1, 0.1, (85, 100)), torch.float64: (0.1, 0.1, (618, 700))}


def itemsize(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def lanes(dtype):
    """Elements of one 16-byte vector of the kernels."""
    return 16 // itemsize(dtype)


def from_bits(dtype, bits):
    size = itemsize(dtype)
    return torch.from_numpy(np.array([bits], dtype=_NP_U[size]).view(_NP_I[size])).view(dtype)[0]


def bits_of(t):
    """The integer view of a contiguous float tensor (writes go through)."""
    return t.view(_INT[t.element_size()])


def other_nan(dtype):
    """A NaN with the sign bit and a payload set: neither the GPU's nor the host's canonical NaN."""
    sign = 1 << (8 * itemsize(dtype) - 1)
    return from_bits(dtype, sign | _INF[dtype] | _QUIET[dtype] | 5)


def ulp_away(x):
    """x one ulp further from zero (the next magnitude up, sign kept)."""
    b = bits_of(x.reshape(1).clone())
    b += 1
    return b.view(x.dtype)[0]


def value_faults(dtype):
    """(name, wanted value, written value, counted) of every value fault of the table."""
    t = lambda v: torch.tensor(v, dtype=dtype)  # noqa: E731
    fi = torch.finfo(dtype)
    sub = from_bits(dtype, 3)
    nan, inf = t(float("nan")), t(float("inf"))
    return [
        ("+1 ulp", t(1.5), ulp_away(t(1.5)), True),
        ("-1 ulp", t(-3.25), ulp_away(t(-3.25)), True),
        ("+0 for -0", t(-0.0), t(0.0), True),
        ("-0 for +0", t(0.0), t(-0.0), True),
        ("subnormal flushed to 0", sub, t(0.0), True),
        ("negative subnormal flushed to -0", -sub, t(-0.0), True),
        ("smallest subnormal flushed to 0", from_bits(dtype, 1), t(0.0), True),
        ("inf for the largest finite", t(fi.max), inf, True),
        ("-inf for the lowest finite", t(fi.min), -inf, True),
        ("largest finite for inf", inf, t(fi.max), True),
        ("finite for NaN", nan, t(1.0), True),
        ("NaN for finite", t(2.0), nan, True),
        ("NaN with another payload", nan, other_nan(dtype), False),
        ("-inf kept", -inf, -inf, False),
    ]


def value_row(dtype, n, seed=0):
    """(want, got, expected, positions): a row of small exact values with every value fault of the table planted at
    its own position (spread over vector lanes), and the number of them that count."""
    g = torch.Generator().manual_seed(seed)
    want = (torch.randint(-64, 65, (n,), generator=g).float() / 8).to(dtype)
    got = want.clone()
    expected, positions = 0, {}
    for k, (name, w, x, counted) in enumerate(value_faults(dtype)):
        i = 3 + 5 * k
        want[i], got[i] = w, x
        positions[name] = i
        expected += counted
    return want, got, expected, positions


def palette(dtype):
    fi = torch.finfo(dtype)
    vals = [0.0, -0.0, fi.max, -fi.max, float("inf"), float("-inf"), float("nan"), 1.0, -2.5, 0.375]
    out = torch.tensor(vals, dtype=torch.float64).to(dtype)
    sub = torch.stack([from_bits(dtype, 1), from_bits(dtype, 7), -from_bits(dtype, 3), torch.tensor(fi.tiny).to(dtype)])
    return torch.cat([out, sub])


def special_step(dtype, rows, n, seed=0):
    """(old, up, dn): a slab and its two neighbour rows drawn from the palette."""
    g = torch.Generator().manual_seed(seed)
    pal = palette(dtype)
    pick = lambda *shape: pal[torch.randint(0, len(pal), shape, generator=g)]  # noqa: E731
    return pick(rows, n).contiguous(), pick(n).contiguous(), pick(n).contiguous()


def special_counts(t):
    """Counts of NaN, inf, -0, +0 and subnormal elements of a field."""
    d = t.double()
    zero = d == 0
    return {"nan": int(torch.isnan(d).sum()), "inf": int(torch.isinf(d).sum()),
            "-0": int((zero & torch.signbit(d)).sum()), "+0": int((zero & ~torch.signbit(d)).sum()),
            "subnormal": int(((d != 0) & (d.abs() < torch.finfo(t.dtype).tiny)).sum())}


def run_field(world, rows, n, dtype, run, checkpoint):
    """The whole closed-form field after the growing or decaying run's checkpoint (0 or 1): (field, steps, alpha, s)."""
    alpha, s, steps = (GROW if run == "grow" else DECAY)[dtype]
    k = steps[checkpoint]
    return reference_steps(initial_field(world, rows, n, dtype), k, alpha, s), k, alpha, s


def assert_run_reaches(field, run, checkpoint):
    """The run's checkpoint holds the values it is there for."""
    c = special_counts(field)
    if run == "grow":   # half is all NaN at the second checkpoint
        assert c["nan"] > 0 and (c["inf"] > 0 or checkpoint == 1), c
    elif checkpoint == 0:
        assert c["subnormal"] > 0 and c["-0"] + c["+0"] > 0, c
    else:
        assert c["-0"] > 0 and c["+0"] > 0 and c["subnormal"] == 0, c
