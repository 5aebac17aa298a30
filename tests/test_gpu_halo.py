"""GPU tests of K-halo (csrc/kernels/halo_stencil.cu): the fused stencil + halo exchange against a plain PyTorch fp32
run of the SAME stencil on the whole undecomposed field.  Virtual ranks (several ranks of one process on one GPU,
peer pointers = plain pointers) exercise the cross-GPU step-word protocol on a 1-GPU box."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SMALL = {"tile_kb": 4, "stages": 6}


def _ring(world, message_bytes, rows, mode, tune=None, **kw):
    from hpc_patterns_b200.models.halo import VirtualRing

    return VirtualRing(world, message_bytes, rows, mode, devices=[0] * world, tune=dict(tune or SMALL), **kw)


def _want(world, rows, row_elems, steps):
    from hpc_patterns_b200.models.halo import initial_field, reference_steps

    return reference_steps(initial_field(world, rows, row_elems), steps)


@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world,rows,message_bytes", [(1, 1, 4096), (1, 3, 20 * 1024 + 16), (2, 1, 64 * 1024),
                                                      (2, 4, 5 * 4096 + 2048), (3, 2, 96 * 1024), (4, 7, 16 * 1024 + 48),
                                                      (8, 2, 40 * 1024)])
def test_virtual_ring_matches_torch(native, mode, world, rows, message_bytes):
    ring = _ring(world, message_bytes, rows, mode)
    try:
        ring.step(5)                                   # one launch per step
        got = ring.gather()
        want = _want(world, rows, message_bytes // 4, 5)
        assert torch.equal(got, want), float((got - want).abs().max())
        for hs in ring.ranks:
            assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
    finally:
        ring.close()


@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world,rows", [(1, 2), (2, 3), (4, 2)])
def test_persistent_multi_step_launch(native, mode, world, rows):
    """k steps in ONE launch per rank: the neighbours' kernels spin on each other's step words while co-resident."""
    message_bytes = 64 * 4096 + 1024
    ring = _ring(world, message_bytes, rows, mode)
    try:
        ring.step(7, persistent=True)
        ring.step(2)                                    # then per-step launches continue the same word sequence
        ring.step(4, persistent=True)
        got = ring.gather()
        want = _want(world, rows, message_bytes // 4, 13)
        assert torch.equal(got, want)
        assert all(hs.launches == 1 + 2 + 1 for hs in ring.ranks)
    finally:
        ring.close()


@pytest.mark.parametrize("mode", ["pull", "push"])
def test_l2_evict_first_hint_is_exact(native, mode):
    """tune l2_hint=1: the slab's own rows stream with an evict_first policy; the values must not change."""
    world, rows, message_bytes = 2, 4, 9 * 4096 + 512
    ring = _ring(world, message_bytes, rows, mode, tune={**SMALL, "l2_hint": 1})
    try:
        ring.step(3)
        ring.step(4, persistent=True)
        assert torch.equal(ring.gather(), _want(world, rows, message_bytes // 4, 7))
    finally:
        ring.close()


def test_default_tiles_large_rows(native):
    """Default 16 KiB x 12 stage geometry, rows larger than one wave of tiles, both modes, single rank."""
    from hpc_patterns_b200.models.halo import HaloStencil
    from hpc_patterns_b200.parallel.comm import Comm

    for mode in ("pull", "push"):
        hs = HaloStencil(Comm(), 0, message_bytes=24 << 20, rows=3, mode=mode)
        try:
            hs.step(3)
            hs.step(1)
            torch.cuda.synchronize()
            hs.check()
            assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
            assert hs.ctas >= torch.cuda.get_device_properties(0).multi_processor_count
        finally:
            hs.close()


@pytest.mark.parametrize("how", ["memcpy", "nccl"])
def test_stock_arm_computes_the_same_time_series(native, how):
    from hpc_patterns_b200.models.halo import HaloStencil
    from hpc_patterns_b200.parallel.comm import Comm

    hs = HaloStencil(Comm(), 0, message_bytes=1 << 20, rows=2, mode="pull", tune=SMALL)
    try:
        for _ in range(3):
            hs.stock_step(how)
        torch.cuda.synchronize()
        assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
        with pytest.raises(RuntimeError, match="reset"):
            hs.step(1)                                  # stock steps never advance the step words of the fused kernel
        hs.reset()
        hs.step(2)
        torch.cuda.synchronize()
        hs.check()
        assert hs.verify_from_init() == 0
    finally:
        hs.close()


def test_unfused_pieces_run(native):
    from hpc_patterns_b200.models.halo import HaloStencil
    from hpc_patterns_b200.parallel.comm import Comm

    hs = HaloStencil(Comm(), 0, message_bytes=1 << 20, rows=2, mode="push", tune=SMALL)
    try:
        hs.compute_only()
        hs.exchange_only()
        torch.cuda.synchronize()
        hs.check()
        hs.reset()
        hs.step(1)
        assert hs.verify_from_init() == 0
    finally:
        hs.close()


def test_dead_neighbour_times_out_instead_of_hanging(native):
    """Rank 0 steps twice while rank 1 never runs: the second step needs rank 1's word -> deadline -> status word."""
    ring = _ring(2, 64 * 1024, 2, "pull", timeout_s=0.2)
    try:
        hs = ring.ranks[0]
        with torch.cuda.stream(ring.streams[0]):
            hs.step(1)
            hs.step(1)
        ring.streams[0].synchronize()
        with pytest.raises(RuntimeError, match="timeout"):
            hs.check()
    finally:
        ring.close()


@pytest.mark.parametrize("world", [1, 2])
def test_step_from_host_round_trip(native, world):
    """Out-of-core stepping: the slab lives in pinned host memory, every step uploads all of it and downloads all of
    the result in column chunks; the halos still travel GPU to GPU."""
    message_bytes, rows, steps = 40 * 4096 + 512, 3, 4
    ring = _ring(world, message_bytes, rows, "push")
    try:
        bufs = [hs.make_host_buffers() for hs in ring.ranks]
        for i in range(steps):
            for hs, b, st in zip(ring.ranks, bufs, ring.streams):
                with torch.cuda.stream(st):
                    hs.step_from_host(b[i & 1], b[(i + 1) & 1], chunks=3)
        want = _want(world, rows, message_bytes // 4, steps)
        got = torch.cat([b[steps & 1] for b in bufs], 0)
        assert torch.equal(got, want)
        assert torch.equal(ring.gather(), want)
        with pytest.raises(RuntimeError, match="reset"):
            ring.ranks[0].step(1)                       # whole-row steps would desynchronise the chunk words
    finally:
        ring.close()


def test_pull_mode_refuses_host_steps(native):
    from hpc_patterns_b200.models.halo import HaloStencil
    from hpc_patterns_b200.parallel.comm import Comm

    hs = HaloStencil(Comm(), 0, message_bytes=1 << 16, rows=1, mode="pull", tune=SMALL)
    try:
        b = hs.make_host_buffers()
        with pytest.raises(RuntimeError, match="push"):
            hs.step_from_host(b[0], b[1])
    finally:
        hs.close()


@pytest.mark.parametrize("rows,row_elems,tune", [(1, 1024, SMALL), (3, 5 * 1024 + 4, SMALL), (8, 1 << 20, None),
                                                 (2, (3 << 20) + 12, {"tile_kb": 32, "stages": 6})])
def test_stencil_step_op_matches_torch_fp32(native, rows, row_elems, tune):
    """The compute half alone, as an op on tensors, against the plain PyTorch fp32 expression (bit-exact)."""
    from hpc_patterns_b200.ops.halo import stencil_step, stencil_step_reference

    g = torch.Generator(device="cuda").manual_seed(3)
    u = torch.randn(rows, row_elems, device="cuda", generator=g)
    lo = torch.randn(row_elems, device="cuda", generator=g)
    hi = torch.randn(row_elems, device="cuda", generator=g)
    for alpha, s in ((0.5, 0.25), (0.3, 0.7)):          # the second pair rounds in every operation
        got = stencil_step(u, lo, hi, alpha=alpha, s=s, tune=tune)
        torch.cuda.synchronize()
        assert torch.equal(got, stencil_step_reference(u, lo, hi, alpha, s))
