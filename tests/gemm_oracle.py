"""Element-wise oracle of the wgmma GEMM kernels (gemm_put.cu, gemm_collective.cu): data and expected values, torch only.

Small dyadic operands (multiples of 1/4 in [-1, 1]) make a GEMM exact, but they set at most the top mantissa bit of a
bf16 value and barely vary the exponent: a kernel that keeps fewer operand or accumulator bits, or truncates where it
should round, still matches them.  The data here uses every mantissa bit the accumulator can afford and is still exact:

* ``exact_operands``      A ``[M, K]`` and B ``[N, K]`` with values +-(1 + m/2^(p-1)) * 2^e, p significant bits, one
                          exponent e per row of A and per row of B.  All products of one output element then lie on the
                          grid g = 2^(e_i + e_j - 2(p-1)) and are smaller than 4 * 2^(e_i + e_j), so with
                          p = ``mantissa_bits(K)`` every partial sum, in any order, is a multiple of g below 2^24 g:
                          exact in fp32.  A GEMM kernel must then reproduce the fp64 product bit for bit.
* ``reference``           that fp64 product (exact on this data, so cuBLAS DGEMM on the GPU is a valid oracle);
                          ``round_bits`` / ``rne_bf16`` the expected bf16 output (round to nearest, ties to even).
* ``bf16_shard_outcomes`` every value a zeroed bf16 shard can hold after P ``red.add.bf16`` additions in any order;
                          ``bf16_shard_bound`` the bound used above four ranks, where the P! orders are too many.
* ``activation_bound``    per-element bounds of the fused epilogue activations against the fp64 activation of the
                          exact C, from the documented error of the approximations the kernel uses.
* ``mlp_exact_operands``  the operands of a relu MLP block whose two chained GEMMs are both exact in fp32 in any order
                          (``mlp_down_bits`` counts the bits of the second one).
* ``general_bound``       a deliberately loose bound for random operands: it admits a truncating fp32 accumulator.
"""
from __future__ import annotations

import itertools
import math
from typing import List, Sequence, Tuple, Union

import torch

FP32_BITS = 24
EXP_RANGE = (-12, 12)           # per-row exponents of exact_operands: products and sums stay normal in fp32
U32 = 2.0 ** -24                # unit roundoff of fp32
TANH_APPROX_REL = 2.0 ** -10.987  # PTX ISA, tanh.approx.f32: maximum relative error
SILU_OVERFLOW = -87.0           # below this, 1 + __expf(-x) exceeds 2^126 and __fdividef may return +-0

Exponents = Union[Tuple[int, int], torch.Tensor]


def mantissa_bits(k: int, extra: int = 0) -> int:
    """Significant bits p of every operand such that a K-term sum (times 2^extra more terms) is exact in fp32:
    sum |a_ik b_jk| < K * 4 * 2^(e_i+e_j) <= 2^(24 - 2(p-1)) * 2^(e_i+e_j) = 2^24 g."""
    return min(8, (FP32_BITS - math.ceil(math.log2(k)) - extra) // 2)


def _row_exponents(rows: int, exps: Exponents, g: torch.Generator, device) -> torch.Tensor:
    if isinstance(exps, torch.Tensor):
        if exps.numel() != rows:
            raise ValueError("one exponent per row")
        return exps.to(device=device, dtype=torch.float64)
    lo, hi = exps
    return torch.randint(lo, hi + 1, (rows,), generator=g, device=device).to(torch.float64)


def _operand(rows: int, k: int, p: int, exps: Exponents, positive: bool, g: torch.Generator,
             device) -> torch.Tensor:
    mant = torch.randint(0, 1 << (p - 1), (rows, k), generator=g, device=device).to(torch.float64)
    sign = torch.randint(0, 2, (rows, k), generator=g, device=device).to(torch.float64) * 2 - 1
    if positive:
        sign = sign.abs()
    e = _row_exponents(rows, exps, g, device)
    return (sign * (1 + mant / (1 << (p - 1))) * torch.exp2(e)[:, None]).to(torch.bfloat16)


def exact_operands(m: int, n: int, k: int, seed: int, *, extra: int = 0, p: int = 0, a_exp: Exponents = EXP_RANGE,
                   b_exp: Exponents = EXP_RANGE, positive: bool = False,
                   device="cpu") -> Tuple[torch.Tensor, torch.Tensor]:
    """bf16 A ``[m, k]`` and B ``[n, k]`` whose product is exact in fp32 in any summation order.

    ``p`` (default ``mantissa_bits(k, extra)``) significant bits per value; ``a_exp`` / ``b_exp`` give the exponent of
    every row, as an inclusive (lo, hi) range to draw from or as one integer per row.  The caller keeps the products
    and results inside the range it wants (the default +-12 keeps everything normal).

    With random signs the partial sums grow like sqrt(K) and use only about 20 of the 24 bits the budget allows for,
    so an accumulator that keeps 21-23 bits still reproduces them.  ``positive`` makes every value positive: the sums
    then grow like K, come within a factor of two of the budget, and need all 24 bits from K = 256 on."""
    p = p or mantissa_bits(k, extra)
    if not 1 <= p <= 8:
        raise ValueError(f"K = {k} leaves no mantissa bit")
    g = torch.Generator(device=device).manual_seed(0x6E440000 + seed)
    return _operand(m, k, p, a_exp, positive, g, device), _operand(n, k, p, b_exp, positive, g, device)


def dyadic_operands(m: int, n: int, k: int, seed: int, device="cpu") -> Tuple[torch.Tensor, torch.Tensor]:
    """The older GEMM tests' data: multiples of 1/4 in [-1, 1] (at most two significant bits)."""
    g = torch.Generator(device=device).manual_seed(seed)
    return tuple((torch.randint(-4, 5, (r, k), generator=g, device=device).float() / 4).to(torch.bfloat16)
                 for r in (m, n))


def reference(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The fp64 product A @ B^T: exact for exact_operands (and for any bf16 data up to K = 2^37)."""
    return a.double() @ b.double().t()


def round_bits(x: torch.Tensor, p: int, mode: str = "rne") -> torch.Tensor:
    """``x`` (fp64) rounded to ``p`` significant bits, without exponent limits: ``rne`` to nearest with ties to even,
    ``trunc`` toward zero.  ``p`` = 8 is bf16, 11 fp16, 24 fp32 (for normal values)."""
    mant, e = torch.frexp(x.double())                  # x = mant * 2^e, |mant| in [0.5, 1)
    scaled = torch.ldexp(mant, torch.full_like(e, p))
    scaled = torch.round(scaled) if mode == "rne" else torch.trunc(scaled)   # torch.round: half to even
    return torch.ldexp(scaled, e - p)


def rne_bf16(x: torch.Tensor) -> torch.Tensor:
    """The bf16 value an fp32 (or exact fp64) result rounds to, to nearest with ties to even."""
    return round_bits(x, 8).to(torch.bfloat16)


def bf16_shard_outcomes(partials: Sequence[torch.Tensor]) -> torch.Tensor:
    """``[P!, ...]`` fp64: every value a zeroed bf16 shard can end up holding after the P additions of
    ``rne_bf16(partials[r])``, one ``red.add.bf16`` per rank, in any order.  Every addition rounds its exact sum
    to bf16 (the hardware may add in fp32 first: with 24 >= 2 * 8 + 2 bits, that double rounding gives the same
    result).  P <= 4 only."""
    if len(partials) > 4:
        raise ValueError("enumerate at most 4! orders; use bf16_shard_bound above")
    x = [round_bits(c, 8) for c in partials]
    out = []
    for order in itertools.permutations(range(len(x))):
        s = torch.zeros_like(x[0])
        for r in order:
            s = round_bits(s + x[r], 8)
        out.append(s)
    return torch.stack(out)


def bf16_shard_bound(partials: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(sum of the rounded partials in fp64, bound): P bf16 additions in any order lie within
    gamma_(P-1) * sum_r |bf16(C_r)| of the exact sum, gamma_k = k u / (1 - k u), with u = 2^-8 the unit roundoff of
    bf16 (8 significant bits).  The tighter (P-1) 2^-9 sum_r |bf16(C_r)| takes half that unit roundoff and is wrong:
    correct orders of 8 ranks reach 0.51 of this bound, beyond that one (test_gemm_oracle.py).  The price of the
    correct bound is that a truncating bf16 conversion stays inside it above four ranks."""
    x = torch.stack([round_bits(c, 8) for c in partials])
    k, u = len(partials) - 1, 2.0 ** -8
    return x.sum(0), k * u / (1 - k * u) * x.abs().sum(0)


def shard_problems(got: torch.Tensor, partials: Sequence[torch.Tensor]) -> str:
    """'' when the bf16 shard ``got`` holds a possible outcome of the additions of ``partials`` in every element."""
    g = got.double()
    if len(partials) <= 4:
        bad = ~(g[None] == bf16_shard_outcomes(partials)).any(0)
        what = "not an outcome of any order of the bf16 additions"
    else:
        ref, bound = bf16_shard_bound(partials)
        bad = ~((g - ref).abs() <= bound)
        what = "outside the bound of the bf16 additions"
    if not bool(bad.any()):
        return ""
    i = tuple(int(v) for v in bad.nonzero()[0])
    return f"{int(bad.sum())} elements {what}, first {i}: got {g[i].item()!r}"


def activation64(c: torch.Tensor, activation: str) -> torch.Tensor:
    """The activations of the fused epilogue, in fp64 (gelu in its tanh form)."""
    c = c.double()
    if activation == "none":
        return c
    if activation == "relu":
        return c.clamp(min=0)
    if activation == "gelu":
        return 0.5 * c * (1 + torch.tanh(math.sqrt(2 / math.pi) * (c + 0.044715 * c ** 3)))
    if activation == "silu":
        return c * torch.sigmoid(c)
    raise ValueError(activation)


def activation_bound(c: torch.Tensor, activation: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """(fp64 activation of the exact accumulator ``c``, per-element bound on the kernel's fp32 result).

    * none, relu: exact (bound 0).
    * gelu: ``0.5 x (1 + t)``, t = ``tanh.approx.f32`` of the fp32 argument.  The approximation errs by at most
      2^-10.987 |t| (PTX ISA); the argument carries at most ~7 fp32 roundings (10 u allowed), which move t by
      |arg| sech^2(arg) times that; both are scaled by 0.5 |x|.  The final add and multiply add 3 ulps of the result
      (and of 0.5 |x| |1 + t| where 1 + t cancels).
    * silu: ``__fdividef(x, 1 + __expf(-x))``.  ``__expf(y)`` errs by at most 2 + floor(1.173 |y|) ulp and
      ``__fdividef`` by 2 ulp for denominators in [2^-126, 2^126] (CUDA C++ Programming Guide, intrinsic functions);
      one more ulp for 1 + e.  Below x = -87 the denominator exceeds 2^126 (or overflows) and the quotient is +-0, so
      the bound there admits 0."""
    x = c.double()
    want = activation64(x, activation)
    if activation in ("none", "relu"):
        return want, torch.zeros_like(want)
    ulp = 2.0 ** -23
    if activation == "gelu":
        arg = math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)
        t = torch.tanh(arg)
        sech2 = torch.minimum(torch.ones_like(arg), 4 * torch.exp(-1.98 * arg.abs()))   # >= sech^2 near arg
        dt = TANH_APPROX_REL * t.abs() + 10 * U32 * arg.abs() * sech2
        bound = 0.5 * x.abs() * (dt + 3 * U32 * (1 + t).abs()) + 3 * ulp * want.abs()
        return want, bound
    if activation == "silu":
        e = torch.exp(-x)
        rel = (2 + torch.floor(1.173 * x.abs())) * ulp * e / (1 + e) + 4 * ulp
        bound = rel * want.abs()
        bound = torch.where(x < SILU_OVERFLOW, want.abs() * (1 + rel), bound)
        return want, bound
    raise ValueError(activation)


def mlp_down_bits(hidden: int, ffn: int, p_up: int, p_down: int) -> int:
    """Bits that the largest partial sum of the second GEMM of a relu MLP block needs on ``mlp_exact_operands`` data.

    Row i of x has exponent e_i and every row of w_up exponent 0, all with ``p_up`` bits: every product of row i of
    the first GEMM is a multiple of g_i = 2^(e_i - 2(p_up-1)) and |C| < 4 hidden 2^e_i.  bf16 keeps such a multiple
    exactly below 2^8 g_i and rounds it to a multiple of 2 g_i or more above, never beyond the power of two above, so
    every hidden value h is a multiple of g_i with |h| / g_i <= 2^(2 + log2 hidden + 2(p_up-1)).  Row n of w_down has
    one exponent d_n over the whole ffn axis and ``p_down`` bits: |w| / 2^(d_n - (p_down-1)) < 2^p_down.  So every
    term h w of output (i, n), on every rank, is a multiple of G = g_i 2^(d_n - (p_down-1)) below 2^(that sum) G, and a
    partial sum of up to ffn terms, in any order and grouping (each rank's K-slice, then the P shard additions), stays
    a multiple of G below 2^bits G: exact in fp32 when bits <= 24."""
    return (math.ceil(math.log2(ffn)) + 2 + math.ceil(math.log2(hidden)) + 2 * (p_up - 1) + p_down)


def mlp_exact_operands(tokens: int, hidden: int, ffn: int, seed: int, *, p_up: int = 2, p_down: int = 3,
                       device="cpu") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """bf16 x ``[tokens, hidden]``, w_up ``[ffn, hidden]``, w_down ``[hidden, ffn]`` of a relu MLP block whose two
    GEMMs are exact in fp32 in any order (``mlp_down_bits`` <= 24): the block output equals the fp64 product of the
    hidden values bit for bit.  Rank r holds rows r of x, row block r of w_up and column block r of w_down.  Exponents
    stay within +-2 per row, so every product and sum is a normal fp32 value."""
    if mlp_down_bits(hidden, ffn, p_up, p_down) > FP32_BITS:
        raise ValueError(f"hidden = {hidden}, ffn = {ffn}, p = {p_up}, {p_down}: the second GEMM needs more than 24 bits")
    x, w_up = exact_operands(tokens, ffn, hidden, seed, p=p_up, a_exp=(-2, 2), b_exp=(0, 0), device=device)
    w_down = exact_operands(hidden, 1, ffn, seed + 1, p=p_down, a_exp=(-2, 2), device=device)[0]
    return x, w_up, w_down


def general_bound(a: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(fp64 product, bound) for any bf16 operands: |C - C64| <= K 2^-22 (|A| |B|^T).  Recursive fp32 summation errs
    by about K 2^-24 |A| |B|^T and a truncating accumulator by K 2^-23; the bound is loose on purpose."""
    k = a.shape[1]
    return reference(a, b), k * 2.0 ** -22 * (a.double().abs() @ b.double().abs().t())


def mismatches(got: torch.Tensor, want: torch.Tensor) -> int:
    """Elements whose values differ (NaN differs from everything; +0 equals -0)."""
    if got.shape != want.shape:
        raise ValueError(f"shapes differ: {tuple(got.shape)} vs {tuple(want.shape)}")
    return int((got.double() != want.double()).sum())


def describe(got: torch.Tensor, want: torch.Tensor) -> str:
    """The first differing elements, for assertion messages."""
    bad = (got.double() != want.double()).nonzero()[:3].tolist()
    return ", ".join(f"{tuple(i)}: got {got[tuple(i)].item()!r} want {want[tuple(i)].item()!r}" for i in bad)
