"""CPU checks of the 16-bit allreduce oracle (tests/lowp_allreduce_oracle.py) and of the bfloat16 / half CLI paths.

* the fact the ring expectations rest on: torch's CPU add on bfloat16 / float16 tensors is the correctly rounded add
  (checked against an exact rounding of the fp64 sum, subnormals, overflow and signed zeros included);
* ``two_shot_expected`` against a plain numpy float32 loop;
* mutations: emulated kernel faults applied to correct results, on the data the GPU tests use -- the comparison those
  tests use must report every one of them, and the miniapp's constant data (rank r holds r) hides all but one;
* ``allreduce.bfloat16`` / ``allreduce.half --cpu`` for every algorithm at 1, 2, 3 and 5 ranks.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from tests.lowp_allreduce_oracle import (FORMAT, LOWP, TORCH_DTYPE, bits, make_inputs, mismatches, ring_expected,
                                         round16, rsag_expected, segment, two_shot_expected)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLD = 5
N = WORLD * 8 * 257                   # 257 vectors per rank slice


def _finite_patterns(rng, n, dtype):
    e_bits, m_bits, _ = FORMAT[dtype]
    raw = rng.integers(0, 1 << 16, n, dtype=np.uint32).astype(np.uint16)
    exp = (raw >> m_bits) & ((1 << e_bits) - 1)
    raw = raw[exp != (1 << e_bits) - 1]                       # finite only
    return torch.from_numpy(raw.view(np.int16).copy()).view(TORCH_DTYPE[dtype])


@pytest.mark.parametrize("dtype", LOWP)
def test_torch_cpu_add_is_the_correctly_rounded_16bit_add(dtype):
    """2^21 random finite bit-pattern pairs, plus pairs near the subnormal range: a + b equals the fp64 sum (exact for
    every pair whose exponents are within 45 of each other; otherwise far below half an ulp) rounded once."""
    rng = np.random.default_rng(1)
    a, b = _finite_patterns(rng, 1 << 21, dtype), _finite_patterns(rng, 1 << 21, dtype)
    m = min(a.numel(), b.numel())
    a, b = a[:m], b[:m]
    sub = make_inputs(2, 1 << 16, dtype, seed=7, kind="subnormal")
    a, b = torch.cat([a, sub[0]]), torch.cat([b, sub[1]])
    want = round16(a.double().numpy() + b.double().numpy(), dtype)
    got = a + b
    assert mismatches(got, want) == 0
    assert bool(torch.isinf(got).any()) and bool(((got != 0) & (got.abs() < torch.finfo(got.dtype).tiny)).any())


@pytest.mark.parametrize("dtype", LOWP)
def test_round16_agrees_with_numpy_float16_and_rz(dtype):
    x = np.random.default_rng(2).standard_normal(1 << 16) * np.exp2(np.random.default_rng(3).integers(-30, 20, 1 << 16))
    x[:4] = [70000.0, -65520.0, 65519.0, 2.0 ** -140]           # past fp16's range, its rounding edge, deep underflow
    r = round16(x, dtype)
    if dtype == "half":
        with np.errstate(over="ignore"):
            assert mismatches(r, torch.from_numpy(x.astype(np.float16))) == 0
    t = round16(x, dtype, "rz")
    assert bool((t.double().abs() <= torch.from_numpy(x).abs()).all()) and bool((t != r).any())
    assert mismatches(round16(t.double().numpy(), dtype, "rz"), t) == 0          # representable values stay


@pytest.mark.parametrize("kind", ["full", "subnormal", "overflow"])
@pytest.mark.parametrize("dtype", LOWP)
def test_two_shot_expected_is_an_fp32_owner_first_loop(dtype, kind):
    if kind == "overflow" and dtype == "bfloat16":
        pytest.skip("the overflow data is fp16's")
    vas = make_inputs(WORLD, N, dtype, seed=11, kind=kind)
    f = [v.float().numpy() for v in vas]
    want = np.empty(N, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(N):
            s = i * WORLD // N
            acc = np.float32(f[s][i])
            for q in range(1, WORLD):
                acc = np.float32(acc + f[(s + q) % WORLD][i])
            want[i] = acc
        assert mismatches(two_shot_expected(vas), round16(want.astype(np.float64), dtype)) == 0


def test_the_data_rounds_and_reaches_the_edges():
    for dtype in LOWP:
        vas = make_inputs(WORLD, N, dtype, seed=1)
        exact = sum(v.double() for v in vas)
        assert mismatches(ring_expected(vas, 0), exact.to(vas[0].dtype)) > N // 5, "sums must round"
        assert not bool(torch.isinf(ring_expected(vas, 0)).any())                                # no overflow
        rank0_first = vas[0].float()
        for v in vas[1:]:
            rank0_first = rank0_first + v.float()
        assert mismatches(two_shot_expected(vas), rank0_first.to(vas[0].dtype)) > N // 100, "the fp32 order shows"
        sub = ring_expected(make_inputs(WORLD, N, dtype, seed=1, kind="subnormal"), 0)
        tiny = torch.finfo(sub.dtype).tiny
        assert int(((sub != 0) & (sub.abs() < tiny)).sum()) > N // 4, "results in the subnormal range"
    ov = ring_expected(make_inputs(WORLD, N, "half", seed=1, kind="overflow"), 2)
    assert int(torch.isinf(ov).sum()) > N // 8 and int(torch.isnan(ov).sum()) > 0
    assert mismatches(torch.full((4,), float("nan"), dtype=torch.half),
                      torch.tensor([0x7E00, 0x7FFF, -1, 0x7C01], dtype=torch.int16).view(torch.half)) == 0


# ------------------------------------------------------------------ mutations ----
def _ring_f32_once(vas, r):
    acc = torch.zeros_like(vas[0], dtype=torch.float32)
    for t in range(len(vas)):
        acc = acc + vas[(r - t) % len(vas)].float()
    return acc.to(vas[0].dtype)


def _ring_last_add_truncated(vas, r, dtype):
    """The ring's result on rank r with its last add (of VA[r+1]) rounded toward zero."""
    world = len(vas)
    acc = torch.zeros_like(vas[0])
    for t in range(world - 1):
        acc = acc + vas[(r - t) % world]
    return round16(acc.double().numpy() + vas[(r + 1) % world].double().numpy(), dtype, "rz")


def _two_shot_rounding_every_add(vas):
    world, n = len(vas), vas[0].numel()
    parts = []
    for s in range(world):
        seg = segment(n, world, s)
        acc = vas[s][seg].clone()
        for q in range(1, world):
            acc = acc + vas[(s + q) % world][seg]
        parts.append(acc)
    return torch.cat(parts)


def _two_shot_rank0_first(vas):
    acc = vas[0].float()
    for v in vas[1:]:
        acc = acc + v.float()
    return acc.to(vas[0].dtype)


def _as_other_format(vas, r):
    other = torch.float16 if vas[0].dtype == torch.bfloat16 else torch.bfloat16
    return ring_expected([v.view(other) for v in vas], r).view(vas[0].dtype)


def _lanes_swapped(t):
    return t.view(torch.int16).view(-1, 2).flip(1).reshape(-1).view(t.dtype)


def _flushed_signed(t):
    tiny = torch.finfo(t.dtype).tiny
    z = torch.where(torch.signbit(t), torch.tensor(-0.0, dtype=t.dtype), torch.tensor(0.0, dtype=t.dtype))
    return torch.where(t.abs() < tiny, z, t)


def _chunk_one_vector_off(t, chunk=8 * 64):
    out = t.clone()
    out[chunk:2 * chunk] = t[chunk + 8:2 * chunk + 8]
    return out


def _mutations(vas, dtype):
    """(name, correct result, faulty result) for every emulated fault, on the data ``vas``."""
    r = 1
    ring = ring_expected(vas, r)
    two = two_shot_expected(vas)
    return [
        ("one add truncates", ring, _ring_last_add_truncated(vas, r, dtype)),
        ("ring partial sums kept in fp32", ring, _ring_f32_once(vas, r)),
        ("two-shot rounds after every add", two, _two_shot_rounding_every_add(vas)),
        ("two-shot sums rank 0 first", two, _two_shot_rank0_first(vas)),
        ("added in the other 16-bit format", ring, _as_other_format(vas, r)),
        ("16-bit lanes of a word swapped", ring, _lanes_swapped(ring)),
        ("subnormal results flushed to zero", ring, _flushed_signed(ring)),
        ("a chunk one vector off", rsag_expected(vas), _chunk_one_vector_off(rsag_expected(vas))),
    ]


@pytest.mark.parametrize("dtype", LOWP)
def test_every_mutation_is_reported_on_the_gpu_data(dtype):
    """The GPU tests' data (full-mantissa and subnormal kinds) and their comparison (``mismatches``) see every fault.
    Faults that only show on some kind of data are caught by the kind the GPU tests run them on."""
    full = make_inputs(WORLD, N, dtype, seed=100 * WORLD)
    sub = make_inputs(WORLD, N, dtype, seed=100 * WORLD, kind="subnormal")
    for (name, want, got), (_, want_s, got_s) in zip(_mutations(full, dtype), _mutations(sub, dtype)):
        seen = mismatches(got, want) + mismatches(got_s, want_s)
        assert seen > 0, f"{dtype}: {name} is not reported"
    # each kind on its own: the subnormal flush needs the subnormal data, everything else shows on full data already
    flags = {name: mismatches(got, want) > 0 for name, want, got in _mutations(full, dtype)}
    assert flags == {name: name != "subnormal results flushed to zero" for name in flags}


@pytest.mark.parametrize("dtype", LOWP)
def test_constant_data_hides_all_but_the_format_error(dtype):
    """Rank r holds r (the miniapps' own check): every partial sum is a small integer, exact in either rounding and
    order, equal in every lane, never subnormal -- only adding the bits in the wrong format changes the result."""
    td = TORCH_DTYPE[dtype]
    vas = [torch.full((N,), float(r), dtype=td) for r in range(WORLD)]
    flags = {name: mismatches(got, want) > 0 for name, want, got in _mutations(vas, dtype)}
    assert flags == {name: name == "added in the other 16-bit format" for name in flags}
    assert bool((ring_expected(vas, 0) == WORLD * (WORLD - 1) / 2).all())
    big = [torch.full((8,), float(r), dtype=td) for r in range(16)]
    for r in range(16):                               # exact up to 16 ranks: every partial sum is an integer <= 120
        assert float(ring_expected(big, r)[0]) == 120.0 and float(two_shot_expected(big)[0]) == 120.0


def test_mismatches_compares_bits_and_nan_classes():
    a = torch.tensor([0.0, 1.0, float("nan"), float("inf")], dtype=torch.bfloat16)
    b = torch.tensor([-0.0, 1.0, float("nan"), float("inf")], dtype=torch.bfloat16)
    assert mismatches(a, b) == 1                      # signed zeros differ, NaNs of any payload agree
    assert bits(a).dtype == torch.int16


# ------------------------------------------------------------ native CLI (--cpu) ----
@pytest.mark.parametrize("algo", ["ring", "ring-unfused", "ring-rsag", "-a"])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
@pytest.mark.parametrize("dtype", LOWP)
def test_cli_cpu_paths(bin_dir, dtype, world, algo, tmp_path):
    rows = tmp_path / "rows.jsonl"
    args = ["-a"] if algo == "-a" else ["--algo", algo]
    p = subprocess.run([os.path.join(bin_dir, f"allreduce.{dtype}"), "--cpu", "-n", str(world), "-p", "12",
                        "--json", str(rows), *args], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == world and f" {dtype} host-threads P={world}" in p.stdout
    import json

    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["type"] == dtype and row["mismatches"] == 0 and row["ranks"] == world


@pytest.mark.parametrize("spelling,name", [("bf16", "bfloat16"), ("float16", "half"), ("fp16", "half"), ("f16", "half")])
def test_cli_type_aliases(bin_dir, spelling, name):
    p = subprocess.run([os.path.join(bin_dir, "allreduce"), "--cpu", "-n", "2", "-p", "8", "--type", spelling],
                       capture_output=True, text=True, timeout=60)
    assert p.returncode == 0 and f" {name} host-threads" in p.stdout, p.stdout + p.stderr
