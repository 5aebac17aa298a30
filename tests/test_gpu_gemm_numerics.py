"""Element-wise numerics of the wgmma GEMM kernels (gemm_put.cu, gemm_collective.cu) on virtual ranks of one GPU.

The older GEMM tests multiply small dyadic operands, which set at most the top mantissa bit of a bf16 value: a kernel
that truncates instead of rounding, keeps fewer operand bits or rounds its partial sums would still pass them.  Here the
operands use every mantissa bit the fp32 accumulator can afford and one exponent per row (tests/gemm_oracle.py), so
every product is still exact, and each output path is compared with the fp64 product:

* A. ``gemm_put``: K/64 in {1, 2, 3, 4, 5, 7, 64}, single CTAs, CTA pairs and the ``cluster=2, ctas=1`` fall-back to a
  single CTA, several tiles per persistent CTA with a tile count that is not a multiple of the grid, tile-row counts
  that are not a multiple of the raster group (5, 12), 1, 3 and 32 tile columns, st and TMA epilogues, fp32 and bf16
  output, local and peer copy (pairwise, not the full product): fp32 bit for bit, bf16 = ``rne_bf16`` of the exact C.
  Every case runs with random signs and with all-positive data: random-sign sums use about 20 of the accumulator's 24
  bits, all-positive ones all 24 from K = 256 on, so an accumulator that keeps fewer bits fails there.
* B. ``gemm_reduce_scatter`` at 1, 2, 3, 5, 6, 8 and 16 ranks, REDG and TMA-reduce epilogues with fp32 shards (bit for
  bit), REDG with bf16 shards (every element one of the outcomes of the P roundings in some order; within the
  summation bound above 4 ranks); two launches with new data, advancing epochs and tickets.
* C. ``gemm_all_to_all`` at 1, 3, 5 and 8 ranks, fp32 and bf16.
* D. ``allgather_gemm`` at 1, 3, 5 and 8 ranks, chunks of 512, 2048 and 4096 bytes, every activation with fp32 and bf16
  output and |C| up to ~150: none and relu exact, gelu and silu within the documented error of the approximations, and
  every bf16 output equal to ``rne_bf16`` of the fp32 output of the same launch configuration.
* The ``cluster=2, ctas=1`` fall-back to a single CTA of the reduce-scatter (REDG, TMA, bf16), the all-to-all and the
  all-gather launchers, on shards that could run as CTA pairs.
* E. random-normal operands with an exponent spread at K = 512, 4096, 16384 through ``gemm_put`` within the general
  bound K 2^-22 |A| |B|^T (sharp for the all-positive variant); the largest error / bound ratio is printed.
* F. subnormal results (every partial product and sum in [2^-149, 2^-126)) on each fp32 output path: every such element
  must be exact, or every one of them +-0 (flushed).  ``SUBNORMALS`` records what each path does on an H100.
"""
import pytest
import torch

from tests.gemm_oracle import (activation_bound, describe, exact_operands, general_bound, mismatches, reference,
                               rne_bf16, shard_problems)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
F32, BF16 = torch.float32, torch.bfloat16
ACT_EXP = dict(a_exp=(-10, 2), b_exp=(-3, 0))     # |C| from below 2^-8 to ~150 at K = 256: past silu's -87
# What each fp32 output path does with a subnormal result (F), as measured on an H100 80GB HBM3: "kept" (exact) or
# "flushed" (+-0).  The tensor cores keep subnormal products and sums; REDG.E.ADD.F32x4.FTZ flushes.
SUBNORMALS = {"put-st": "kept", "put-tma": "kept", "rs-red": "flushed", "rs-tma": "kept"}


@pytest.fixture(scope="module")
def native():
    import hpc_patterns_b200

    assert torch.cuda.is_available()
    torch.cuda.set_device(DEV)
    return hpc_patterns_b200.native()


def _exact(m, n, k, seed, **kw):
    return exact_operands(m, n, k, seed, device=DEV, **kw)


def _nan(*shape, dtype=F32):
    return torch.full(shape, float("nan"), device=DEV, dtype=dtype)


def _expected(c64, dtype):
    return c64.float() if dtype == F32 else rne_bf16(c64)


# ---- A. gemm_put --------------------------------------------------------------------------------------------------
# (K/64, cluster, ctas, epilogue, out, copies, tile rows, tile columns).  cluster 2 with ctas 1 is the fall-back to a
# single CTA.  Every other grid leaves >= 3 tiles per CTA and does not divide the tile count.
PUT_CASES = [
    (1, 1, 4, "st", F32, "both", 5, 3), (1, 1, 50, "tma", BF16, "peer", 5, 32),
    (1, 2, 10, "st", BF16, "local", 12, 3), (1, 2, 14, "tma", F32, "both", 2, 32),
    (3, 1, 10, "st", BF16, "peer", 12, 3), (3, 1, 4, "tma", F32, "local", 5, 3),
    (3, 2, 6, "st", F32, "peer", 4, 5), (3, 2, 8, "tma", BF16, "both", 12, 3),
    (5, 1, 50, "st", F32, "local", 5, 32), (5, 1, 4, "tma", BF16, "both", 5, 3),
    (5, 2, 14, "st", BF16, "both", 2, 32), (5, 2, 10, "tma", F32, "peer", 12, 3),
    (2, 2, 1, "st", F32, "both", 12, 1), (4, 2, 1, "tma", BF16, "local", 4, 1),
    (7, 1, 4, "st", BF16, "both", 5, 3), (7, 2, 10, "tma", F32, "both", 12, 3),
    (64, 2, 98, "st", F32, "both", 12, 32), (64, 1, 4, "tma", BF16, "peer", 5, 3),
    (64, 2, 1, "tma", F32, "peer", 2, 3),
]


def _put_id(case):
    kb, cl, ctas, epi, out, copies, tm, tn = case
    return f"kb{kb}-c{cl}x{ctas}-{epi}-{'f32' if out == F32 else 'bf16'}-{copies}-{tm}x{tn}"


@pytest.mark.parametrize("positive", [False, True], ids=["signed", "positive"])
@pytest.mark.parametrize("case", PUT_CASES, ids=[_put_id(c) for c in PUT_CASES])
def test_gemm_put_exact(native, case, positive):
    """Signed data sees an accumulator of about 20 bits or fewer; all-positive data needs all 24 from K = 256 on."""
    from hpc_patterns_b200.ops.gemm import gemm_put

    kb, cluster, ctas, epilogue, out, copies, tm, tn = case
    m, n, k = 128 * tm, 256 * tn, 64 * kb
    a, b = _exact(m, n, k, seed=kb * 100 + tm * 10 + tn, positive=positive)
    c_local = _nan(m, n, dtype=out) if copies != "peer" else None
    c_peer = _nan(m, n, dtype=out) if copies != "local" else 0
    launched = gemm_put(a, b, c_local, c_peer, ctas=ctas, cluster=cluster, out_dtype=out, epilogue=epilogue)
    torch.cuda.synchronize()
    assert launched == (ctas & ~1 if cluster == 2 and ctas > 1 else ctas)
    want = _expected(reference(a, b), out)
    for name, c in (("local", c_local), ("peer", c_peer)):
        if isinstance(c, torch.Tensor):
            assert mismatches(c, want) == 0, f"{name}: {mismatches(c, want)} elements differ: {describe(c, want)}"


# ---- B. gemm_reduce_scatter ---------------------------------------------------------------------------------------
RS_WORLDS = [1, 2, 3, 5, 6, 8, 16]
SHARD_TILES = {1: 3, 2: 2, 3: 1, 5: 1, 6: 2, 8: 1, 16: 1}      # 2 and 6 ranks: CTA pairs (auto)


@pytest.mark.parametrize("variant", ["red", "tma", "red-bf16"])
@pytest.mark.parametrize("world", RS_WORLDS)
def test_gemm_reduce_scatter_exact(native, world, variant):
    """The P partial sums of one product with P*K terms, so the fp32 sum is exact in any order."""
    from hpc_patterns_b200.ops.gemm import gemm_reduce_scatter

    out = BF16 if variant.endswith("bf16") else F32
    m, n, k = 128 * world * SHARD_TILES[world], 512, 64 * (1 + world % 4)
    pads = [torch.zeros(256, dtype=torch.int32, device=DEV) for _ in range(world)]
    issued = [0] * world
    for epoch in (1, 2):
        a, b = _exact(m, n, world * k, seed=epoch * 100 + world)
        a_r = [a[:, r * k:(r + 1) * k].contiguous() for r in range(world)]
        b_r = [b[:, r * k:(r + 1) * k].contiguous() for r in range(world)]
        shards = [torch.zeros(m // world, n, device=DEV, dtype=out) for _ in range(world)]
        for r in range(world):
            done = [pads[q].data_ptr() + 4 * (native.PAD_DONE + r) for q in range(world)]
            issued[r] += gemm_reduce_scatter(a_r[r], b_r[r], shards, r, done_flags=done, done_epoch=epoch,
                                             ticket=pads[r].data_ptr() + 4 * native.PAD_LOCAL, ticket_base=issued[r],
                                             ctas=0 if epoch == 1 else 3, out_dtype=out, epilogue=variant[:3])
        for q in range(world):
            native.wait_flags(pads[q].data_ptr() + 4 * native.PAD_DONE, world, epoch, int(5e9), 0,
                              torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got = torch.cat(shards, 0)
        if out == F32:
            want = reference(a, b).float()
            assert mismatches(got, want) == 0, f"epoch {epoch}: {describe(got, want)}"
        else:
            problem = shard_problems(got, [reference(a_r[r], b_r[r]) for r in range(world)])
            assert problem == "", f"epoch {epoch}: {problem}"
        for q in range(world):
            assert pads[q][native.PAD_DONE:native.PAD_DONE + world].tolist() == [epoch] * world
            assert int(pads[q][native.PAD_LOCAL]) == issued[q]


# ---- C. gemm_all_to_all -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("world", [1, 3, 5, 8])
def test_gemm_all_to_all_exact(native, world, out):
    from hpc_patterns_b200.ops.gemm import gemm_all_to_all

    rows = 128 * (2 if world == 3 else 1)
    m, n, k = rows * world, 768, 192
    ops = [_exact(m, n, k, seed=300 + 10 * world + r) for r in range(world)]
    recv = [_nan(world, rows, n, dtype=out) for _ in range(world)]
    for r in range(world):
        gemm_all_to_all(*ops[r], recv, r, out_dtype=out, ctas=4)
    torch.cuda.synchronize()
    for r in range(world):
        want = _expected(reference(*ops[r]), out)
        for q in range(world):
            got, block = recv[q][r], want[q * rows:(q + 1) * rows]
            assert mismatches(got, block) == 0, f"recv[{q}][{r}]: {describe(got, block)}"


# ---- D. allgather_gemm --------------------------------------------------------------------------------------------
ACTIVATIONS = ["none", "relu", "gelu", "silu"]


@pytest.mark.parametrize("world,chunk", [(1, 4096), (3, 512), (5, 2048), (8, 4096), (5, 512), (3, 2048)])
def test_allgather_gemm_exact_and_activations(native, world, chunk):
    from hpc_patterns_b200.ops.gemm import allgather_gemm

    rows = 128 * (2 if world < 5 else 1)
    m, n, k = rows * world, 512, 256
    a, _ = _exact(m, 256, k, seed=400 + world, **ACT_EXP)
    bs = [_exact(256, n, k, seed=500 + 10 * world + r, **ACT_EXP)[1] for r in range(world)]
    src = [a[q * rows:(q + 1) * rows] for q in range(world)]
    status = torch.zeros(world, dtype=torch.int32, device=DEV)
    for r in range(world):
        c64 = reference(a, bs[r])
        assert float(c64.min()) < -87 and float(c64.max()) > 87
        for act in ACTIVATIONS:
            got = {}
            for out in (F32, BF16):
                a_full = _nan(m, k, dtype=BF16)
                a_full[r * rows:(r + 1) * rows] = src[r]
                ready = torch.zeros(m // 128, dtype=torch.int32, device=DEV)
                got[out] = _nan(m, n, dtype=out)
                allgather_gemm(a_full, src, bs[r], got[out], r, ready=ready, chunk_bytes=chunk, timeout_ns=int(5e9),
                               status=status.data_ptr() + 4 * r, ctas=7, activation=act)
                torch.cuda.synchronize()
                assert torch.equal(a_full, a), f"rank {r}: gathered A differs"
            want, bound = activation_bound(c64, act)
            err = (got[F32].double() - want).abs()
            bad = ~(err <= bound)
            assert not bool(bad.any()), (f"rank {r} {act}: {int(bad.sum())} elements outside the bound, worst "
                                         f"{float(((err - bound) / want.abs().clamp(min=1e-30)).max())} relative")
            assert mismatches(got[BF16], rne_bf16(got[F32].double())) == 0, \
                f"rank {r} {act}: bf16 output is not the rounded fp32 output: {describe(got[BF16], got[F32])}"
    assert status.tolist() == [0] * world


@pytest.mark.parametrize("launcher", ["rs-red", "rs-tma", "rs-bf16", "a2a", "ag"])
def test_collective_cta_pair_fallback(native, launcher):
    """``cluster=2`` with ``ctas=1`` on shards that could run as CTA pairs: every launcher falls back to one single
    CTA (the whole 256-row B box instead of the pair's half) that walks all tiles, and the result stays exact."""
    from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_all_to_all, gemm_reduce_scatter

    world, rows, n, k = 2, 256, 512, 192                 # two tile rows per shard: pairable
    m = world * rows
    if launcher.startswith("rs"):
        out = BF16 if launcher == "rs-bf16" else F32
        a, b = _exact(m, n, world * k, seed=600)
        a_r = [a[:, r * k:(r + 1) * k].contiguous() for r in range(world)]
        b_r = [b[:, r * k:(r + 1) * k].contiguous() for r in range(world)]
        shards = [torch.zeros(rows, n, device=DEV, dtype=out) for _ in range(world)]
        for r in range(world):
            assert gemm_reduce_scatter(a_r[r], b_r[r], shards, r, ctas=1, cluster=2, out_dtype=out,
                                       epilogue=launcher[3:] if out == F32 else "red") == 1
        torch.cuda.synchronize()
        got = torch.cat(shards, 0)
        if out == F32:
            want = reference(a, b).float()
            assert mismatches(got, want) == 0, describe(got, want)
        else:
            problem = shard_problems(got, [reference(a_r[r], b_r[r]) for r in range(world)])
            assert problem == "", problem
    elif launcher == "a2a":
        ops = [_exact(m, n, k, seed=610 + r) for r in range(world)]
        recv = [_nan(world, rows, n) for _ in range(world)]
        for r in range(world):
            assert gemm_all_to_all(*ops[r], recv, r, ctas=1, cluster=2) == 1
        torch.cuda.synchronize()
        for r in range(world):
            want = reference(*ops[r]).float()
            for q in range(world):
                got, block = recv[q][r], want[q * rows:(q + 1) * rows]
                assert mismatches(got, block) == 0, f"recv[{q}][{r}]: {describe(got, block)}"
    else:
        a, b = _exact(m, n, k, seed=620)
        src = [a[q * rows:(q + 1) * rows] for q in range(world)]
        status = torch.zeros(world, dtype=torch.int32, device=DEV)
        want = reference(a, b).float()
        for r in range(world):
            a_full = _nan(m, k, dtype=BF16)
            a_full[r * rows:(r + 1) * rows] = src[r]
            c = _nan(m, n)
            ready = torch.zeros(m // 128, dtype=torch.int32, device=DEV)
            assert allgather_gemm(a_full, src, b, c, r, ready=ready, timeout_ns=int(5e9),
                                  status=status.data_ptr() + 4 * r, ctas=1, cluster=2) == 1
            torch.cuda.synchronize()
            assert torch.equal(a_full, a), f"rank {r}: gathered A differs"
            assert mismatches(c, want) == 0, f"rank {r}: {describe(c, want)}"
        assert status.tolist() == [0] * world


# ---- E. general data ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("positive", [False, True], ids=["signed", "positive"])
@pytest.mark.parametrize("k", [512, 4096, 16384])
def test_gemm_put_general_data_within_bound(native, k, positive):
    """The largest error / bound ratio is printed; ``pytest -s`` or ``-rP`` shows it
    (``-k general_data -m gpu -rP``)."""
    from hpc_patterns_b200.ops.gemm import gemm_put

    g = torch.Generator(device=DEV).manual_seed(k + positive)

    def operand(rows):
        x = torch.randn(rows, k, device=DEV, generator=g)
        x = x * torch.exp2(torch.randint(-6, 7, (rows, k), device=DEV, generator=g).float())
        return (x.abs() if positive else x).to(BF16)

    a, b = operand(256), operand(512)
    c = _nan(256, 512)
    gemm_put(a, b, c, 0, ctas=3)
    torch.cuda.synchronize()
    ref, bound = general_bound(a, b)
    ratio = float(((c.double() - ref).abs() / bound).max())
    print(f"\ngeneral data K={k} {'positive' if positive else 'signed'}: max |C - C64| / bound = {ratio:.3e}")
    assert ratio <= 1.0


# ---- F. subnormal results -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(SUBNORMALS))
def test_subnormal_results(native, path):
    """Even rows of A: exponent -68, every B row: -67, so every product, partial and full sum of those rows lies in
    [2^-149, 2^-126) on the 2^-149 grid (K = 64 per rank, 2 ranks for the reduce-scatter).  Odd rows stay normal."""
    from hpc_patterns_b200.ops.gemm import gemm_put, gemm_reduce_scatter

    m, n, k = 256, 256, 64
    world = 2 if path.startswith("rs") else 1
    a_exp = torch.where(torch.arange(m) % 2 == 0, -68, 53)
    a, b = _exact(m, n, world * k, seed=7, p=8, a_exp=a_exp, b_exp=torch.full((n,), -67))
    want = reference(a, b)
    if world == 1:
        got = _nan(m, n)
        gemm_put(a, b, got, 0, ctas=1, epilogue=path[4:])
    else:
        shards = [torch.zeros(m // world, n, device=DEV) for _ in range(world)]
        for r in range(world):
            gemm_reduce_scatter(a[:, r * k:(r + 1) * k].contiguous(), b[:, r * k:(r + 1) * k].contiguous(), shards, r,
                                epilogue=path[3:])
        torch.cuda.synchronize()
        got = torch.cat(shards, 0)
    torch.cuda.synchronize()
    sub = (want.abs() < 2.0 ** -126) & (want != 0)
    assert int(sub.sum()) > m * n // 3 and float(want[sub].abs().min()) >= 2.0 ** -149
    assert mismatches(got[~sub], want[~sub].float()) == 0, "a normal result differs"
    kept = mismatches(got[sub], want[sub].float()) == 0
    flushed = bool((got[sub] == 0).all())
    seen = "kept" if kept else "flushed" if flushed else "mixed"
    print(f"\nsubnormal results on {path}: {seen}")
    assert seen == SUBNORMALS[path]
