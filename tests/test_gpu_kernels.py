"""Single-GPU numerics tests: every sm_90a kernel against a plain PyTorch reference."""

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _stream():
    return torch.cuda.current_stream(0).cuda_stream


@pytest.mark.parametrize("engine", ["ldst", "tma"])
@pytest.mark.parametrize("nbytes", [1024, 65536 + 16, (1 << 20) + 48, 1000003, 64 << 20])
def test_copy_matches_torch(native, dev, engine, nbytes):
    src = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device=dev)
    dst = torch.zeros(nbytes + 64, dtype=torch.uint8, device=dev)
    ctas = native.copy(dst.data_ptr(), src.data_ptr(), nbytes, False, engine, {}, {}, 0, _stream())
    torch.cuda.synchronize()
    assert ctas >= 1
    assert torch.equal(dst[:nbytes], src)
    assert int(dst[nbytes:].sum()) == 0  # no overrun


@pytest.mark.parametrize("unroll", [1, 2, 4, 8])
def test_copy_ldst_unroll_variants(native, dev, unroll):
    n = (8 << 20) + 32
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev)
    dst = torch.zeros(n, dtype=torch.uint8, device=dev)
    native.copy(dst.data_ptr(), src.data_ptr(), n, True, "ldst", {"unroll": unroll, "ctas": 37}, {}, 0, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst, src)


@pytest.mark.parametrize("tune", [{"vec_bytes": 32}, {"vec_bytes": 32, "blocked": 1, "ctas": 53},
                                  {"blocked": 1, "threads": 1024, "unroll": 8}, {"vec_bytes": 32, "unroll": 8}])
@pytest.mark.parametrize("n", [(8 << 20) + 32, 1000003, 4096])
def test_copy_ldst_wide_and_blocked(native, dev, tune, n):
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev)
    dst = torch.zeros(n + 64, dtype=torch.uint8, device=dev)
    native.copy(dst.data_ptr(), src.data_ptr(), n, False, "ldst", tune, {}, 0, _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst[:n], src) and int(dst[n:].sum()) == 0


@pytest.mark.parametrize("stages,stage_kb", [(2, 8), (4, 16), (8, 16), (6, 32)])
def test_copy_tma_stage_variants(native, dev, stages, stage_kb):
    n = (24 << 20) + 4096 + 16
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev)
    dst = torch.zeros(n, dtype=torch.uint8, device=dev)
    native.copy(dst.data_ptr(), src.data_ptr(), n, False, "tma", {"stages": stages, "stage_kb": stage_kb}, {}, 0,
                _stream())
    torch.cuda.synchronize()
    assert torch.equal(dst, src)


def test_copy_signal_and_wait_roundtrip(native, dev):
    """Epilogue signal (last CTA publishes) + a waiting kernel + prologue wait, on one GPU."""
    pad = torch.zeros(256, dtype=torch.int32, device=dev)
    n = 4 << 20
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev)
    dst = torch.zeros(n, dtype=torch.uint8, device=dev)
    flag = pad.data_ptr() + 4 * native.PAD_DONE
    ticket = pad.data_ptr() + 4 * native.PAD_LOCAL
    status = pad.data_ptr() + 4 * 200
    issued = 0
    for epoch in (1, 2, 3):
        sync = {"signal_flag": flag, "signal_epoch": epoch, "ticket": ticket, "ticket_base": issued,
                "timeout_ns": int(5e9), "status": status}
        issued += native.copy(dst.data_ptr(), src.data_ptr(), n, False, "ldst", {}, sync, 0, _stream())
        native.wait(flag, epoch, int(5e9), status, _stream())
        torch.cuda.synchronize()
        assert int(pad[native.PAD_DONE].item()) == epoch
        assert int(pad[native.PAD_LOCAL].item()) == issued
        assert int(pad[200].item()) == native.STATUS_OK
    assert torch.equal(dst, src)


def test_wait_timeout_sets_status_instead_of_hanging(native, dev):
    pad = torch.zeros(64, dtype=torch.int32, device=dev)
    native.wait(pad.data_ptr(), 5, int(2e7), pad.data_ptr() + 4 * 8, _stream())  # 20 ms deadline
    torch.cuda.synchronize()
    assert int(pad[8].item()) & 0xFFFFFFFF == native.STATUS_TIMEOUT


def test_fill_and_verify_pattern(native, dev):
    from hpc_patterns_b200.ops.p2p import pattern_reference

    n = 1 << 20
    buf = torch.zeros(n, dtype=torch.int32, device=dev)
    native.fill_pattern(buf.data_ptr(), n, 0xDEADBEEF, _stream())
    torch.cuda.synchronize()
    ref = pattern_reference(n, 0xDEADBEEF)
    got = buf.cpu().to(torch.int64) & 0xFFFFFFFF
    assert torch.equal(got, ref)
    counters = torch.zeros(2, dtype=torch.int64, device=dev)
    native.verify_pattern(buf.data_ptr(), n, 0xDEADBEEF, counters.data_ptr(), counters.data_ptr() + 8)
    torch.cuda.synchronize()
    assert int(counters[0]) == 0 and int(counters[1]) == int(ref.sum())
    buf[12345] ^= 1
    counters.zero_()
    native.verify_pattern(buf.data_ptr(), n, 0xDEADBEEF, counters.data_ptr(), counters.data_ptr() + 8)
    torch.cuda.synchronize()
    assert int(counters[0]) == 1


def test_fill_triad_inputs_and_verify(native, dev):
    from hpc_patterns_b200.ops.fused import triad_inputs_reference

    n = 1 << 18
    b = torch.zeros(n, device=dev)
    c = torch.zeros(n, device=dev)
    native.fill_triad_inputs(b.data_ptr(), c.data_ptr(), n, 3, _stream())
    torch.cuda.synchronize()
    rb, rc = triad_inputs_reference(n, 3)
    assert torch.equal(b.cpu(), rb) and torch.equal(c.cpu(), rc)
    a = (rb + 3.0 * rc).to(dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    native.verify_triad(a.data_ptr(), n, 3, 3.0, cnt.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert int(cnt) == 0
    a[77] += 1
    native.verify_triad(a.data_ptr(), n, 3, 3.0, cnt.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert int(cnt) == 1


@pytest.mark.parametrize("ratio", [1, 3])
def test_fused_exchange_loopback(native, ratio):
    from hpc_patterns_b200.models.peer2pear import FusedTriadExchange
    from hpc_patterns_b200.parallel.comm import Comm

    for engine in ("ldst", "tma"):
        ex = FusedTriadExchange(Comm(), 0, nbytes=8 << 20, engine=engine, compute_ratio=ratio)
        for _ in range(3):
            ex.step()
        torch.cuda.synchronize()
        ex.check()
        assert ex.verify() == 0
        assert torch.equal(ex.a, ex.b + 3.0 * ex.c)
        host = ex.make_host_input()
        assert ex.step_from_host(host, chunks=4) == 0
        ex.close()


def test_busy_wait_semantics(native, dev):
    out = torch.full((300,), -1.0, device=dev)
    native.busy_wait(out.data_ptr(), 300, 3, _stream())
    torch.cuda.synchronize()
    assert float(out[0]) == 0.0          # y=0 stays 0 through the FMA chain
    assert bool(torch.isinf(out[1:]).all())  # everything else overflows to +inf


def test_fused_bench_pinned_host_copy(native, dev):
    n = 1 << 20
    h = torch.randn(n).pin_memory()
    d = torch.zeros(n, device=dev)
    back = torch.zeros(n).pin_memory()
    native.fused_bench([{"kind": "copy", "n": n, "dst": d.data_ptr(), "src": h.data_ptr()}], "tma", {}, 0, _stream())
    native.fused_bench([{"kind": "copy", "n": n, "dst": back.data_ptr(), "src": d.data_ptr()}], "tma", {}, 0, _stream())
    torch.cuda.synchronize()
    assert torch.equal(d.cpu(), h) and torch.equal(back, h)


@pytest.mark.parametrize("dtype,td", [("double", torch.float64), ("long", torch.int64), ("ulong", torch.int64),
                                      ("short", torch.int16), ("ushort", torch.int16), ("uchar", torch.uint8),
                                      ("uint", torch.int32), ("float", torch.float32), ("int", torch.int32)])
def test_accumulate_every_reference_datatype_matches_torch(native, dev, dtype, td):
    """VC += VA for every type the reference's datatype trait maps to an MPI_SUM type (mpi_datatype.hpp:28-51), random
    data incl. wrap-around for the integers, against the PyTorch add of the bit-identical dtype; odd tail included."""
    n = (1 << 16) + 3
    g = torch.Generator(device=dev).manual_seed(7)
    if td.is_floating_point:
        va = torch.randn(n, dtype=td, device=dev, generator=g)
        vc = torch.randn(n, dtype=td, device=dev, generator=g)
    else:
        info = torch.iinfo(td)
        va = torch.randint(info.min, info.max, (n,), dtype=torch.int64, device=dev, generator=g).to(td)
        vc = torch.randint(info.min, info.max, (n,), dtype=torch.int64, device=dev, generator=g).to(td)
    want = vc + va                      # integer adds wrap in torch as they do in two's complement
    native.accumulate(va.data_ptr(), vc.data_ptr(), n, dtype, _stream())
    torch.cuda.synchronize()
    assert torch.equal(vc, want)


@pytest.mark.parametrize("dtype,td", [("float", torch.float32), ("int", torch.int32), ("double", torch.float64),
                                      ("long", torch.int64), ("short", torch.int16), ("uchar", torch.uint8)])
def test_allreduce_building_blocks(native, dev, dtype, td):
    n = (1 << 18) + 4
    va = torch.zeros(n, dtype=td, device=dev)
    vb = torch.zeros(n, dtype=td, device=dev)
    vc = torch.zeros(n, dtype=td, device=dev)
    native.init3(va.data_ptr(), vb.data_ptr(), vc.data_ptr(), n, 5, 7, 1, dtype, _stream())
    native.accumulate(va.data_ptr(), vc.data_ptr(), n, dtype, _stream())
    native.accumulate(vb.data_ptr(), vc.data_ptr(), n, dtype, _stream())
    torch.cuda.synchronize()
    assert torch.equal(vc, torch.full((n,), 13, dtype=td, device=dev))
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    native.count_mismatch(vc.data_ptr(), n, 13.0, dtype, cnt.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert int(cnt) == 0
    vc[5] = 12
    native.count_mismatch(vc.data_ptr(), n, 13.0, dtype, cnt.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert int(cnt) == 1


@pytest.mark.parametrize("algo", ["ring", "ring-unfused", "twoshot", "nccl"])
@pytest.mark.parametrize("dtype", ["float", "int", "double", "short"])
def test_allreduce_miniapp_single_rank(native, algo, dtype):
    from hpc_patterns_b200.models.allreduce import AllreduceMiniapp
    from hpc_patterns_b200.parallel.comm import Comm

    app = AllreduceMiniapp(Comm(), 0, log2_elems=16, dtype=dtype, algo=algo)
    res = app.run(iters=2, warmup=1)
    app.close()
    assert res.mismatches == 0 and res.ms > 0


@pytest.mark.parametrize("mode", ["serial", "in_order", "out_of_order", "host_threads", "nowait", "fused"])
def test_concurency_cuda_backend_all_modes(native, mode):
    rc, out, err = native.concurency_main(
        [mode, "--repetitions", "3", "--globalsize_default_memory", "4000000",
         "--commands", "C", "D2D", "--commands", "H2D", "D2H", "--commands", "C", "A", "--commands", "M2D", "C"],
        "cuda")
    assert out.count("## " + mode) == 4, out + err
    assert "Parameters used:" in out and "tripcount_C" in out
    assert rc in (0, 1)


def test_concurency_bench_api_profiling(native):
    r = native.concurency_bench("cuda", "serial", ["C", "DH"], {"globalsize_C": 1, "tripcount_C": 2000,
                                                                "globalsize_DH": 1 << 20}, True, -1, 3, False)
    assert len(r["per_command_us"]) == 2 and len(r["device_us"]) == 2
    assert all(t > 0 for t in r["device_us"])
    r2 = native.concurency_bench("cuda", "in_order", ["C", "DH"], {"globalsize_C": 1, "tripcount_C": 2000,
                                                                   "globalsize_DH": 1 << 20}, True, -1, 3, False)
    assert r2["device_total_us"] > 0


def test_smoke_entry():
    import __graft_entry__ as g

    g.smoke()


@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("tripcount,ctas", [(1, 2), (3, 6), (100, 148)])
def test_tcgen05_tile_loop_matches_reference(native, dev, tripcount, ctas, cluster):
    """T command: out[cta] = tripcount * (A . B^T) with bf16 operands, fp32 register accumulation (wgmma)."""
    ops = torch.zeros(native.tc_busy_operand_bytes() // 2, dtype=torch.bfloat16, device=dev)
    per = native.tc_busy_out_elems_per_cta()
    out = torch.full((ctas * per,), float("nan"), device=dev)
    native.tc_fill_operands(ops.data_ptr(), _stream())
    native.tc_busy(ops.data_ptr(), out.data_ptr(), ctas, tripcount, _stream(), cluster)
    torch.cuda.synchronize()
    a = ops[:128 * 64].view(128, 64).float()
    b = ops[128 * 64:].view(256, 64).float()
    # plain PyTorch fp32 reference of the same op
    ref = tripcount * (a @ b.t())
    got = out.view(ctas, 128, 256)
    assert torch.equal(got[0], ref), (got[0] - ref).abs().max()
    assert bool((got == got[0]).all())
    assert float(a.abs().max()) == 1.0 and float(b.abs().max()) == 2.0


def test_tcgen05_duration_scales_with_tripcount(native, dev):
    ops = torch.zeros(native.tc_busy_operand_bytes() // 2, dtype=torch.bfloat16, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    out = torch.zeros(sms * native.tc_busy_out_elems_per_cta(), device=dev)
    native.tc_fill_operands(ops.data_ptr(), _stream())

    def run(tc):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        native.tc_busy(ops.data_ptr(), out.data_ptr(), sms, tc, _stream())
        torch.cuda.synchronize()
        e0.record()
        native.tc_busy(ops.data_ptr(), out.data_ptr(), sms, tc, _stream())
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    t1, t2 = run(20000), run(40000)
    assert 1.6 < t2 / t1 < 2.4, (t1, t2)
    flops = sms * 40000 * 2.0 * 128 * 256 * 64
    print(f"wgmma tile loop: {flops / (t2 * 1e-3) / 1e12:.0f} TFLOP/s bf16 over {sms} CTAs")


def test_concurency_tensor_command(native):
    rc, out, err = native.concurency_main(["nowait", "--repetitions", "3", "--globalsize_default_memory", "8000000",
                                           "--commands", "T", "H2D", "--commands", "T", "C"], "cuda")
    assert out.count("## nowait | T") == 2, out + err
    assert "tripcount_T" in out


@pytest.mark.parametrize("cluster", [1, 0])
@pytest.mark.parametrize("m,n,k", [(128, 256, 64), (256, 512, 256), (1024, 1024, 512), (384, 768, 4096),
                                   (2048, 2048, 1024), (1280, 512, 192)])
def test_gemm_put_matches_fp32_reference(native, dev, m, n, k, cluster):
    """wgmma GEMM (TMA ring, register accumulators) vs a plain PyTorch fp32 matmul; loop-back 'peer'."""
    from hpc_patterns_b200.ops.gemm import gemm_put, gemm_reference

    torch.manual_seed(m + n + k)
    a = (torch.randint(-4, 5, (m, k), device=dev).float() / 4).to(torch.bfloat16)   # exactly representable
    b = (torch.randint(-4, 5, (n, k), device=dev).float() / 4).to(torch.bfloat16)
    c_local = torch.full((m, n), float("nan"), device=dev)
    c_peer = torch.full((m, n), float("nan"), device=dev)
    ctas = gemm_put(a, b, c_local, c_peer, cluster=cluster)
    torch.cuda.synchronize()
    ref = gemm_reference(a, b)
    assert ctas >= 1
    assert torch.equal(c_local, ref), float((c_local - ref).abs().max())   # sums of small dyadic rationals: exact
    assert torch.equal(c_peer, c_local)
    # random normal data: compare with tolerance against the fp32 reference
    a = torch.randn(m, k, device=dev).to(torch.bfloat16)
    b = torch.randn(n, k, device=dev).to(torch.bfloat16)
    gemm_put(a, b, c_local, 0, cluster=cluster)
    torch.cuda.synchronize()
    ref = gemm_reference(a, b)
    assert torch.allclose(c_local, ref, rtol=1e-3, atol=1e-2 * (k ** 0.5)), float((c_local - ref).abs().max())
    # bf16 output: the fp32 accumulator rounded once
    c_bf = torch.zeros(m, n, device=dev, dtype=torch.bfloat16)
    gemm_put(a, b, c_bf, 0, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.equal(c_bf, c_local.to(torch.bfloat16))


def test_gemm_put_signal_and_few_ctas(native, dev):
    from hpc_patterns_b200.ops.gemm import gemm_put, gemm_reference

    a = (torch.randint(-2, 3, (512, 256), device=dev).float()).to(torch.bfloat16)
    b = (torch.randint(-2, 3, (1024, 256), device=dev).float()).to(torch.bfloat16)
    c_peer = torch.zeros(512, 1024, device=dev)
    pad = torch.zeros(256, dtype=torch.int32, device=dev)
    sync = {"signal_flag": pad.data_ptr() + 4 * native.PAD_DONE, "signal_epoch": 7,
            "ticket": pad.data_ptr() + 4 * native.PAD_LOCAL, "ticket_base": 0}
    ctas = gemm_put(a, b, None, c_peer, sync=sync, ctas=3, cluster=1)   # 16 tiles on 3 persistent CTAs
    torch.cuda.synchronize()
    assert ctas == 3 and int(pad[native.PAD_DONE]) == 7 and int(pad[native.PAD_LOCAL]) == 3
    assert torch.equal(c_peer, gemm_reference(a, b))
    c_peer.zero_()
    sync.update(signal_epoch=8, ticket_base=3)
    ctas = gemm_put(a, b, None, c_peer, sync=sync, ctas=5, cluster=2)   # CTA pairs: 5 -> 4 CTAs
    torch.cuda.synchronize()
    assert ctas == 4 and int(pad[native.PAD_DONE]) == 8 and int(pad[native.PAD_LOCAL]) == 7
    assert torch.equal(c_peer, gemm_reference(a, b))


@pytest.mark.parametrize("m,n,k", [(256, 256, 64), (256, 512, 256), (1024, 1024, 512), (2048, 2048, 1024),
                                   (512, 768, 4096), (8192, 8192, 512)])
def test_gemm_put_cta_pairs_exact(native, dev, m, n, k):
    """CTA pairs sharing the B tile through TMA multicast (`cluster=2`): exact against the fp32 reference (inputs are
    multiples of 1/4, sums are exact), local and 'peer' copy, fp32 and bf16 output."""
    from hpc_patterns_b200.ops.gemm import gemm_put, gemm_reference

    torch.manual_seed(m + n + k)
    a = (torch.randint(-4, 5, (m, k), device=dev).float() / 4).to(torch.bfloat16)
    b = (torch.randint(-4, 5, (n, k), device=dev).float() / 4).to(torch.bfloat16)
    c_local = torch.full((m, n), float("nan"), device=dev)
    c_peer = torch.full((m, n), float("nan"), device=dev)
    ctas = gemm_put(a, b, c_local, c_peer, cluster=2)
    torch.cuda.synchronize()
    ref = gemm_reference(a, b)
    assert ctas >= 2 and ctas % 2 == 0
    assert torch.equal(c_local, ref), float((c_local - ref).abs().max())
    assert torch.equal(c_peer, c_local)
    c_bf = torch.zeros(m, n, device=dev, dtype=torch.bfloat16)
    gemm_put(a, b, c_bf, 0, out_dtype=torch.bfloat16, cluster=2, ctas=6)   # several tiles per pair
    torch.cuda.synchronize()
    assert torch.equal(c_bf, ref.to(torch.bfloat16))
