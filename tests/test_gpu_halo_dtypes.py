"""GPU tests of K-halo's double, bfloat16 and half fields (the double, __nv_bfloat16 and __half instantiations of
halo_stencil_kernel, halo_init_kernel, halo_verify_init_kernel and halo_verify_step_kernel in
csrc/kernels/halo_stencil.cu), bit for bit against models/halo.py::reference_steps: virtual rings of 1-8 ranks in pull
and push mode with per-step and persistent launches, rows that are not a multiple of the column tile, 24 MiB rows at
the default geometry, the stock memcpy / NCCL arms, step_from_host, the stencil_step op (subnormal results of the
16-bit types are kept), and the native and torchrun command lines."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float64, torch.bfloat16, torch.float16]
IDS = ["double", "bfloat16", "half"]


def _ring(world, message_bytes, rows, mode, dtype, tune, per_step=2, persistent=3, alpha=0.5, s=0.25):
    from hpc_patterns_b200.models.halo import VirtualRing, initial_field, reference_steps

    ring = VirtualRing(world, message_bytes, rows, mode, devices=[0] * world, tune=dict(tune), dtype=dtype,
                       alpha=alpha, s=s)
    try:
        ring.step(per_step)
        ring.step(persistent, persistent=True)
        got = ring.gather()
        n = message_bytes // got.element_size()
        want = reference_steps(initial_field(world, rows, n, dtype), per_step + persistent, alpha, s)
        assert got.dtype == dtype and torch.equal(got, want), float((got.double() - want.double()).abs().max())
        for hs in ring.ranks:
            assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
    finally:
        ring.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("rows", [1, 2, 3, 7])
def test_virtual_ring(native, dtype, mode, world, rows):
    """3 column tiles of 4 KiB and a ragged fourth one of 48 bytes; two per-step launches, then one persistent one."""
    _ring(world, 3 * 4096 + 48, rows, mode, dtype, {"tile_kb": 4})


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("mode", ["pull", "push"])
def test_other_coefficients_and_tall_slab(native, dtype, mode):
    _ring(3, 5 * 2048 + 16, 13, mode, dtype, {"tile_kb": 2}, alpha=0.3, s=0.7)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("mode", ["pull", "push"])
def test_large_rows_default_geometry(native, dtype, mode):
    _ring(2, 24 << 20, 3, mode, dtype, {}, per_step=1, persistent=2)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("how", ["memcpy", "nccl"])
def test_stock_steps(native, dtype, how):
    """The stock arm (kernel, wait, library transfer, wait) on one rank: the same time series as the fused step."""
    from hpc_patterns_b200.models.halo import VirtualRing, initial_field, reference_steps

    ring = VirtualRing(1, 4 * 4096 + 32, 3, "pull", devices=[0], tune={"tile_kb": 4}, dtype=dtype)
    try:
        hs = ring.ranks[0]
        for _ in range(4):
            hs.stock_step(how)
        torch.cuda.synchronize()
        want = reference_steps(initial_field(1, 3, hs.row_elems, dtype), 4)
        assert torch.equal(hs.u_tensor().cpu(), want)
        assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
    finally:
        ring.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_step_from_host(native, dtype):
    from hpc_patterns_b200.models.halo import VirtualRing, initial_field, reference_steps

    message_bytes, rows, steps = 40 * 1024 + 16, 3, 3
    ring = VirtualRing(2, message_bytes, rows, "push", devices=[0, 0], tune={"tile_kb": 1}, dtype=dtype)
    try:
        bufs = [hs.make_host_buffers() for hs in ring.ranks]
        assert bufs[0][0].dtype == dtype
        for i in range(steps):
            for hs, b in zip(ring.ranks, bufs):
                hs.step_from_host(b[i & 1], b[(i + 1) & 1])
        got = torch.cat([b[steps & 1] for b in bufs], 0)
        assert torch.equal(got, reference_steps(initial_field(2, rows, ring.ranks[0].row_elems, dtype), steps))
    finally:
        ring.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("rows", [1, 2, 8, 13])
def test_stencil_step_random(native, dtype, rows):
    from hpc_patterns_b200.ops.halo import stencil_step, stencil_step_reference

    g = torch.Generator(device="cuda").manual_seed(rows)
    row_elems = 9 * 1024 + 8
    u, lo, hi = (torch.randn(shape, device="cuda", generator=g, dtype=torch.float64).to(dtype)
                 for shape in ((rows, row_elems), (row_elems,), (row_elems,)))
    got = stencil_step(u, lo, hi, alpha=0.3, s=0.7)
    torch.cuda.synchronize()
    assert got.dtype == dtype and torch.equal(got, stencil_step_reference(u, lo, hi, 0.3, 0.7))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bfloat16", "half"])
def test_stencil_step_keeps_subnormals(native, dtype):
    """Inputs a few steps above the smallest subnormal of the type: many results are subnormal and must not be flushed."""
    from hpc_patterns_b200.ops.halo import stencil_step, stencil_step_reference

    tiny = torch.finfo(dtype).smallest_normal
    g = torch.Generator(device="cuda").manual_seed(7)
    row_elems = 4096
    u, lo, hi = ((torch.randint(-64, 65, shape, device="cuda", generator=g).double() * (tiny / 64)).to(dtype)
                 for shape in ((4, row_elems), (row_elems,), (row_elems,)))
    want = stencil_step_reference(u, lo, hi, 0.3, 0.7)
    sub = (want != 0) & (want.abs() < tiny)
    assert int(sub.sum()) > 1000
    got = stencil_step(u, lo, hi, alpha=0.3, s=0.7)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_stencil_step_rejects_mixed_dtypes(native):
    from hpc_patterns_b200.ops.halo import stencil_step

    u = torch.zeros(2, 64, device="cuda", dtype=torch.bfloat16)
    row = torch.zeros(64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="one dtype"):
        stencil_step(u, row.half(), row)
    with pytest.raises(ValueError, match="one dtype"):
        stencil_step(u, row, row, out=torch.empty(2, 64, device="cuda"))
    with pytest.raises(ValueError, match="16 bytes"):
        stencil_step(torch.zeros(2, 4, device="cuda", dtype=torch.float16), row[:4].half(), row[:4].half())


@pytest.mark.parametrize("cmd", [["halo.bfloat16", "-n", "4"], ["halo", "--type", "double", "-n", "2", "--per-step"],
                                 ["halo.half", "-n", "3", "--mode", "push"]], ids=["bf16", "double-per-step", "half-push"])
def test_native_cli(bin_dir, cmd):
    ranks = int(cmd[cmd.index("-n") + 1])
    p = subprocess.run([os.path.join(bin_dir, cmd[0]), *cmd[1:], "--bytes", str(8 << 20), "--rows", "3", "--steps", "6",
                        "--iters", "2"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    # rank threads print their lines concurrently, so they may interleave: count them
    assert p.stdout.count("Passed") == ranks and "FAILED" not in p.stdout, p.stdout
    want = {"halo.bfloat16": "bfloat16", "halo": "double", "halo.half": "half"}[cmd[0]]
    assert f"type={want}" in p.stdout


def test_torchrun_front_door(native):
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr",
           "127.0.0.1", "--master-port", "29653", "-m", "hpc_patterns_b200", "halo", "--type", "half", "--bytes",
           str(8 << 20), "--rows", "3", "--steps", "5", "--iters", "2"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "Passed 0" in p.stdout and "type=half" in p.stdout
