"""GPU tests of the two GEMM kernels that carry their collective (csrc/kernels/gemm_collective.cu).

One-GPU tests emulate P ranks with P launches on the
same device ("virtual ranks": every rank's shard / row block is a separate buffer, peer pointers are plain local
pointers), which exercises the whole tile order, ownership, gather and signalling logic without NVLink.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    import hpc_patterns_b200

    return hpc_patterns_b200.native()


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _dyadic(shape, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randint(-4, 5, shape, device=dev, generator=g).float() / 4).to(torch.bfloat16)


@pytest.mark.parametrize("world,m,n,k,cluster", [(1, 256, 256, 64, 1), (2, 512, 512, 256, 1), (2, 1024, 512, 128, 2),
                                                 (4, 2048, 1024, 256, 0), (8, 2048, 768, 512, 0),
                                                 (4, 8192, 2048, 256, 0), (2, 2048, 512, 128, 2),
                                                 (4, 4096, 1024, 512, 2)])
@pytest.mark.parametrize("epilogue", ["red", "tma"])
def test_gemm_reduce_scatter_virtual_ranks(native, dev, world, m, n, k, cluster, epilogue):
    """Every virtual rank adds its partial product into the owners' shards; the shards must hold the exact sum
    (operands are small dyadic rationals, so fp32 addition is exact in any order)."""
    from hpc_patterns_b200.ops.gemm import gemm_reduce_scatter, gemm_reference

    a = [_dyadic((m, k), dev, 10 + r) for r in range(world)]
    b = [_dyadic((n, k), dev, 50 + r) for r in range(world)]
    shards = [torch.zeros(m // world, n, device=dev) for _ in range(world)]
    pads = [torch.zeros(256, dtype=torch.int32, device=dev) for _ in range(world)]   # one signal pad per rank
    issued = [0] * world
    for epoch in (1, 2):                                   # twice: tickets and epochs count up
        for s in shards:
            s.zero_()
        for r in range(world):
            done = [pads[q].data_ptr() + 4 * (native.PAD_DONE + r) for q in range(world)]
            ctas = gemm_reduce_scatter(a[r], b[r], shards, r, done_flags=done, done_epoch=epoch,
                                       ticket=pads[r].data_ptr() + 4 * native.PAD_LOCAL, ticket_base=issued[r],
                                       cluster=cluster, ctas=0 if epoch == 1 else 6, epilogue=epilogue)
            issued[r] += ctas
        for q in range(world):
            native.wait_flags(pads[q].data_ptr() + 4 * native.PAD_DONE, world, epoch, int(5e9), 0,
                              torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        ref = sum(gemm_reference(a[r], b[r]) for r in range(world))
        got = torch.cat(shards, 0)
        assert torch.equal(got, ref), float((got - ref).abs().max())
        for q in range(world):
            assert pads[q][native.PAD_DONE:native.PAD_DONE + world].tolist() == [epoch] * world


@pytest.mark.parametrize("m,n,k,cluster", [(128, 256, 64, 1), (512, 768, 256, 1), (2048, 1024, 512, 0), (1024, 512, 128, 2),
                                           (1024, 1024, 256, 2)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_gemm_put_tma_store_epilogue(native, dev, m, n, k, cluster, out_dtype):
    """gemm_put with the C tile leaving through the TMA unit (swizzled smem pieces + UTMASTG) instead of st.global:
    same bits as the fp32 reference, local and 'peer' copy."""
    from hpc_patterns_b200.ops.gemm import gemm_put, gemm_reference

    a = _dyadic((m, k), dev, 1)
    b = _dyadic((n, k), dev, 2)
    c_local = torch.full((m, n), float("nan"), device=dev, dtype=out_dtype)
    c_peer = torch.full((m, n), float("nan"), device=dev, dtype=out_dtype)
    pad = torch.zeros(256, dtype=torch.int32, device=dev)
    sync = {"signal_flag": pad.data_ptr() + 4 * native.PAD_DONE, "signal_epoch": 5,
            "ticket": pad.data_ptr() + 4 * native.PAD_LOCAL, "ticket_base": 0}
    ctas = gemm_put(a, b, c_local, c_peer, sync=sync, out_dtype=out_dtype, cluster=cluster, epilogue="tma")
    torch.cuda.synchronize()
    ref = gemm_reference(a, b).to(out_dtype)
    assert torch.equal(c_local, ref) and torch.equal(c_peer, ref)
    assert int(pad[native.PAD_DONE]) == 5 and int(pad[native.PAD_LOCAL]) == ctas
    c_peer.fill_(float("nan"))
    gemm_put(a, b, None, c_peer, out_dtype=out_dtype, cluster=cluster, ctas=4, epilogue="tma")   # few persistent CTAs
    torch.cuda.synchronize()
    assert torch.equal(c_peer, ref)


@pytest.mark.parametrize("world,m,n,k,cluster", [(2, 512, 256, 64, 1), (4, 2048, 512, 64, 0)])
def test_gemm_reduce_scatter_bf16_shards(native, dev, world, m, n, k, cluster):
    """bf16 shards (REDG.E.ADD.BF16x8).  Ternary operands and K = 64: every partial sum and every running total is an
    integer of magnitude <= 256, exactly representable in bf16, so the result is exact in any order."""
    from hpc_patterns_b200.ops.gemm import gemm_reduce_scatter, gemm_reference

    g = torch.Generator(device=dev).manual_seed(3)
    a = [torch.randint(-1, 2, (m, k), device=dev, generator=g).to(torch.bfloat16) for _ in range(world)]
    b = [torch.randint(-1, 2, (n, k), device=dev, generator=g).to(torch.bfloat16) for _ in range(world)]
    shards = [torch.zeros(m // world, n, device=dev, dtype=torch.bfloat16) for _ in range(world)]
    for r in range(world):
        gemm_reduce_scatter(a[r], b[r], shards, r, cluster=cluster, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    ref = sum(gemm_reference(a[r], b[r]) for r in range(world))
    assert torch.equal(torch.cat(shards, 0).float(), ref)


@pytest.mark.parametrize("world,m,n,k,cluster", [(1, 128, 256, 64, 1), (2, 512, 256, 128, 1), (4, 2048, 512, 256, 0),
                                                 (8, 2048, 768, 128, 2)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_gemm_all_to_all_virtual_ranks(native, dev, world, m, n, k, cluster, out_dtype):
    """recv[q][r] must hold row block q of rank r's product."""
    from hpc_patterns_b200.ops.gemm import gemm_all_to_all, gemm_reference

    rows = m // world
    a = [_dyadic((m, k), dev, 20 + r) for r in range(world)]
    b = [_dyadic((n, k), dev, 60 + r) for r in range(world)]
    recv = [torch.full((world, rows, n), float("nan"), device=dev, dtype=out_dtype) for _ in range(world)]
    for r in range(world):
        gemm_all_to_all(a[r], b[r], recv, r, out_dtype=out_dtype, cluster=cluster)
    torch.cuda.synchronize()
    for r in range(world):
        ref = gemm_reference(a[r], b[r]).to(out_dtype)
        for q in range(world):
            assert torch.equal(recv[q][r], ref[q * rows:(q + 1) * rows]), (q, r)


@pytest.mark.parametrize("world,m,n,k,cluster,chunk", [(1, 256, 256, 64, 1, 0), (2, 512, 256, 128, 1, 0),
                                                       (2, 1024, 512, 256, 2, 2048), (4, 2048, 512, 512, 0, 0),
                                                       (8, 2048, 256, 1024, 0, 1024), (4, 4096, 1024, 2048, 0, 4096),
                                                       (2, 2048, 512, 256, 2, 0), (4, 4096, 512, 1024, 2, 2048)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_allgather_gemm_virtual_ranks(native, dev, world, m, n, k, cluster, chunk, out_dtype):
    """Every virtual rank gathers the other ranks' row blocks while it multiplies; its C must equal the product
    with the whole A and its gathered buffer must hold the whole A."""
    from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_reference

    rows = m // world
    a = _dyadic((m, k), dev, 7)
    b = [_dyadic((n, k), dev, 90 + r) for r in range(world)]
    a_full = [torch.full((m, k), float("nan"), device=dev, dtype=torch.bfloat16) for _ in range(world)]
    ready = [torch.zeros(m // 128, dtype=torch.int32, device=dev) for _ in range(world)]
    status = torch.zeros(world, dtype=torch.int32, device=dev)
    per_launch = native.allgather_gemm_chunks_per_block(k, chunk)
    for it in range(2):                                    # twice: the arrival counters count up
        for r in range(world):
            a_full[r].fill_(float("nan"))
            a_full[r][r * rows:(r + 1) * rows] = a[r * rows:(r + 1) * rows]
        torch.cuda.synchronize()
        c = [torch.full((m, n), float("nan"), device=dev, dtype=out_dtype) for _ in range(world)]
        for r in range(world):
            src = [a_full[q][q * rows:(q + 1) * rows] for q in range(world)]
            allgather_gemm(a_full[r], src, b[r], c[r], r, ready=ready[r], ready_base=it * per_launch,
                           chunk_bytes=chunk, timeout_ns=int(5e9), status=status.data_ptr() + 4 * r,
                           cluster=cluster, ctas=0 if it == 0 else 10)
        torch.cuda.synchronize()
        assert status.tolist() == [0] * world
        for r in range(world):
            assert torch.equal(a_full[r], a), f"rank {r}: gathered A differs"
            ref = gemm_reference(a, b[r])
            assert torch.equal(c[r], ref.to(out_dtype)), float((c[r].float() - ref).abs().max())
            if world > 1:
                want = [(it + 1) * per_launch if blk // (rows // 128) != r else 0 for blk in range(m // 128)]
                assert ready[r].tolist() == want


@pytest.mark.parametrize("activation", ["relu", "gelu", "silu"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_allgather_gemm_fused_activation(native, dev, activation, out_dtype):
    """The activation runs on the fp32 accumulator in the epilogue: relu is exact, gelu (tanh form, tanh.approx) and
    silu (__expf) are compared with the PyTorch fp32 functions within the approximations' error."""
    from hpc_patterns_b200.models.tensor_parallel import apply_activation
    from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_reference

    world, m, n, k = 2, 512, 512, 128
    rows = m // world
    a = _dyadic((m, k), dev, 11)
    b = _dyadic((n, k), dev, 12)
    for r in range(world):
        a_full = torch.zeros(m, k, device=dev, dtype=torch.bfloat16)
        a_full[r * rows:(r + 1) * rows] = a[r * rows:(r + 1) * rows]
        ready = torch.zeros(m // 128, dtype=torch.int32, device=dev)
        c = torch.full((m, n), float("nan"), device=dev, dtype=out_dtype)
        allgather_gemm(a_full, [a[q * rows:(q + 1) * rows] for q in range(world)], b, c, r, ready=ready,
                       timeout_ns=int(5e9), activation=activation)
        torch.cuda.synchronize()
        ref = apply_activation(gemm_reference(a, b), activation)
        if activation == "relu":
            assert torch.equal(c, ref.to(out_dtype))
        else:
            tol = 2e-2 if out_dtype == torch.bfloat16 else 2e-3
            assert torch.allclose(c.float(), ref, rtol=tol, atol=tol), float((c.float() - ref).abs().max())


def test_all_to_all_then_gemm_is_the_same_kernel(native, dev):
    """Dispatch -> GEMM: rank r's A is slot r of every rank's send buffer [P, M/P, K] — allgather_gemm with
    a_src[q] = send_q[r] (the sources are arbitrary row-block pointers)."""
    from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_reference

    world, m, n, k = 4, 2048, 256, 256
    rows = m // world
    send = [_dyadic((world, rows, k), dev, 30 + q) for q in range(world)]
    b = [_dyadic((n, k), dev, 70 + r) for r in range(world)]
    status = torch.zeros(world, dtype=torch.int32, device=dev)
    for r in range(world):
        a_full = torch.full((m, k), float("nan"), device=dev, dtype=torch.bfloat16)
        a_full[r * rows:(r + 1) * rows] = send[r][r]                       # my own contribution is local
        ready = torch.zeros(m // 128, dtype=torch.int32, device=dev)
        c = torch.zeros(m, n, device=dev)
        allgather_gemm(a_full, [send[q][r] for q in range(world)], b[r], c, r, ready=ready, timeout_ns=int(5e9),
                       status=status.data_ptr() + 4 * r)
        torch.cuda.synchronize()
        a_ref = torch.cat([send[q][r] for q in range(world)], 0)
        assert torch.equal(a_full, a_ref) and torch.equal(c, gemm_reference(a_ref, b[r]))
    assert status.tolist() == [0] * world


def test_allgather_gemm_reports_a_missing_block(native, dev):
    """A block that never arrives must end in a timeout status, not in a hang: ready_base is set one launch too
    high, so the counters can never reach the target."""
    from hpc_patterns_b200.ops.gemm import allgather_gemm

    m, n, k, world = 512, 256, 128, 2
    a_full = torch.zeros(m, k, device=dev, dtype=torch.bfloat16)
    b = torch.zeros(n, k, device=dev, dtype=torch.bfloat16)
    c = torch.zeros(m, n, device=dev)
    ready = torch.zeros(m // 128, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    src = [a_full[:256], a_full[256:]]
    allgather_gemm(a_full, src, b, c, 0, ready=ready, ready_base=native.allgather_gemm_chunks_per_block(k, 0),
                   timeout_ns=int(2e8), status=status.data_ptr())
    torch.cuda.synchronize()
    assert int(status[0]) & 0xFFFFFFFF == native.STATUS_TIMEOUT


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_tensor_parallel_layers_torchrun():
    n = min(torch.cuda.device_count(), 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr",
           "127.0.0.1", "--master-port", "29641", os.path.join(ROOT, "scripts", "tp_bench.py"), "--check",
           "--tokens", "2048", "--out-features", "1024", "--in-features", "1024", "--steps", "3"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    assert '"row_parallel_exact": true' in p.stdout and '"column_parallel_exact": true' in p.stdout
    assert '"row_parallel_allreduce_exact": false' not in p.stdout      # absent when the box has no NVLS multicast
