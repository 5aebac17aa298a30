"""GPU tests of the K-halo kernel's register data path (csrc/kernels/halo_stencil.cu, ownership in halo_columns.h) in
the cases the other halo tests do not reach: slabs taller than the rows one column keeps in flight (R = 13, 31), one
CTA, more CTAs than a launch has column tiles, 1 KiB tiles (most threads of a CTA own no column), a row whose last
tile holds a single float4, persistent launches on 1-3 virtual ranks in pull and push mode, and mode `none`.
Exact against plain PyTorch fp32."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run_ring(world, message_bytes, rows, mode, tune, steps=(3, 4)):
    from hpc_patterns_b200.models.halo import VirtualRing, initial_field, reference_steps

    ring = VirtualRing(world, message_bytes, rows, mode, devices=[0] * world, tune=dict(tune))
    try:
        ring.step(steps[0])
        ring.step(steps[1], persistent=True)
        got = ring.gather()
        want = reference_steps(initial_field(world, rows, message_bytes // 4), sum(steps))
        assert torch.equal(got, want), float((got - want).abs().max())
        for hs in ring.ranks:
            assert hs.verify_last_step() == 0
    finally:
        ring.close()


@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("rows", [13, 31])
def test_tall_slabs(native, rows, world, mode):
    """More interior rows than one chunk of loads in flight; a ragged last tile."""
    _run_ring(world, 21 * 4096 + 272, rows, mode, {"tile_kb": 4})


@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("tune,message_bytes", [
    ({"ctas": 1}, 9 * 16384 + 4096),                  # one CTA walks every tile
    ({"tile_kb": 1}, 37 * 1024 + 512),               # 64 float4 per tile: 448 of 512 threads idle
    ({"tile_kb": 2}, 11 * 2048 + 16),                # the last tile holds a single float4
    ({"tile_kb": 1, "ctas": 5}, 23 * 1024 + 16),     # ragged CTA share and a one-float4 tile
], ids=["ctas1", "tile1", "last-float4", "tile1-ctas5"])
@pytest.mark.parametrize("world", [1, 3])
def test_geometry_edges(native, world, mode, tune, message_bytes):
    _run_ring(world, message_bytes, 8, mode, tune)


@pytest.mark.parametrize("rows", [1, 2, 8, 13])
def test_more_ctas_than_tiles_in_host_chunks(native, rows):
    """step_from_host launches 16 column chunks of 2-3 tiles with the whole row's grid: most CTAs own no tile."""
    from hpc_patterns_b200.models.halo import VirtualRing, initial_field, reference_steps

    message_bytes, steps = 40 * 1024 + 16, 3
    ring = VirtualRing(2, message_bytes, rows, "push", devices=[0, 0], tune={"tile_kb": 1})
    try:
        assert ring.ranks[0].ctas > 3
        bufs = [hs.make_host_buffers() for hs in ring.ranks]
        for i in range(steps):
            for hs, b in zip(ring.ranks, bufs):
                hs.step_from_host(b[i & 1], b[(i + 1) & 1])
        got = torch.cat([b[steps & 1] for b in bufs], 0)
        assert torch.equal(got, reference_steps(initial_field(2, rows, message_bytes // 4), steps))
    finally:
        ring.close()


@pytest.mark.parametrize("tune", [None, {"tile_kb": 1}, {"ctas": 1}], ids=["default", "tile1", "ctas1"])
@pytest.mark.parametrize("rows", [1, 7, 13, 31])
def test_none_mode_tall_slabs(native, rows, tune):
    from hpc_patterns_b200.ops.halo import stencil_step, stencil_step_reference

    g = torch.Generator(device="cuda").manual_seed(rows)
    row_elems = 9 * 1024 + 4
    u = torch.randn(rows, row_elems, device="cuda", generator=g)
    lo = torch.randn(row_elems, device="cuda", generator=g)
    hi = torch.randn(row_elems, device="cuda", generator=g)
    got = stencil_step(u, lo, hi, alpha=0.3, s=0.7, tune=tune)
    torch.cuda.synchronize()
    assert torch.equal(got, stencil_step_reference(u, lo, hi, 0.3, 0.7))
