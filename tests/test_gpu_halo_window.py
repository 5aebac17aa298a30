"""GPU tests of the K-halo kernel's boundary-first load order and register row window (csrc/kernels/halo_stencil.cu)
at the slab heights where the order has its special cases (R = 1, 2, 3), on rings of 1 to 3 virtual ranks, in all three
modes, and at the default geometry.  Exact against plain PyTorch fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SMALL = {"tile_kb": 4, "stages": 6}


def _ring(world, message_bytes, rows, mode, tune):
    from hpc_patterns_b200.models.halo import VirtualRing

    return VirtualRing(world, message_bytes, rows, mode, devices=[0] * world, tune=dict(tune))


def _want(world, rows, row_elems, steps):
    from hpc_patterns_b200.models.halo import initial_field, reference_steps

    return reference_steps(initial_field(world, rows, row_elems), steps)


@pytest.mark.parametrize("tune", [SMALL, {}, {"tile_kb": 8, "stages": 3}, {"tile_kb": 32, "stages": 7, "out_stages": 2}],
                         ids=["small", "default", "min-ring", "tile32"])
@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("rows", [1, 2, 3])
def test_short_slabs_match_torch(native, rows, world, mode, tune):
    """Per-step launches, then one persistent launch; a ragged last column tile in every row."""
    message_bytes = 37 * 4096 + 272
    ring = _ring(world, message_bytes, rows, mode, tune)
    try:
        ring.step(3)
        ring.step(4, persistent=True)
        got = ring.gather()
        assert torch.equal(got, _want(world, rows, message_bytes // 4, 7)), float((got - _want(
            world, rows, message_bytes // 4, 7)).abs().max())
        for hs in ring.ranks:
            assert hs.verify_last_step() == 0
    finally:
        ring.close()


@pytest.mark.parametrize("rows", [1, 2, 3, 8])
@pytest.mark.parametrize("tune", [None, SMALL], ids=["default", "small"])
def test_none_mode_step_op_matches_torch(native, rows, tune):
    """Mode `none` (local halo buffers) through the stencil op."""
    from hpc_patterns_b200.ops.halo import stencil_step, stencil_step_reference

    g = torch.Generator(device="cuda").manual_seed(rows)
    row_elems = 70 * 1024 + 8
    u = torch.randn(rows, row_elems, device="cuda", generator=g)
    lo = torch.randn(row_elems, device="cuda", generator=g)
    hi = torch.randn(row_elems, device="cuda", generator=g)
    got = stencil_step(u, lo, hi, alpha=0.3, s=0.7, tune=tune)
    torch.cuda.synchronize()
    assert torch.equal(got, stencil_step_reference(u, lo, hi, 0.3, 0.7))


def test_default_geometry_bench_rows(native):
    """The default geometry at the benchmark's slab height over many column tiles per CTA, pull and push."""
    from hpc_patterns_b200.models.halo import HaloStencil
    from hpc_patterns_b200.parallel.comm import Comm

    for mode in ("pull", "push"):
        hs = HaloStencil(Comm(), 0, message_bytes=(40 << 20) + 4096, rows=8, mode=mode)
        try:
            hs.step(2)
            hs.step(3)
            torch.cuda.synchronize()
            hs.check()
            assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
        finally:
            hs.close()
