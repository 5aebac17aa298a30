"""One process per rank on the CPU box: the flagship's process-per-GPU path (torchrun's shape) over `gloo` and the
emulated device of tests/emu_device.py::SharedEmuNative.

Buffers live in named shared-memory segments that the ranks hand each other through the same `ipc_export` / all-gather /
`ipc_open` sequence CUDA IPC handles take on the GPU box (parallel/symmetric.py), waits spin with a deadline, and the
ranks really run concurrently: a persistent multi-step launch of rank 0 advances only as fast as rank 1 publishes its
step words.  What this covers that the single-process emulation cannot: `SymmetricBuffer`'s multi-process constructor,
`SignalPads.device_barrier` across processes, `Comm` reductions inside `BlockTimer`, K steps in one launch against a
neighbour in another process, the stock arm through `torch.distributed` send/recv, and `bench.py` at N = 2 — the JSON
line of a multi-rank run with the world > 1 branches (NVLink roofline term, NCCL-arm fields, silent non-zero ranks)."""
import io
import json
import os
import sys
import traceback

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ring_job(comm, emu, mode):
    from hpc_patterns_b200.models.halo import HaloStencil, initial_field, reference_steps

    rows, n = 3, 2048 + 64
    hs = HaloStencil(comm, comm.device, 4 * n, rows, mode, tune={"tile_kb": 1}, timeout_s=20.0)
    hs.step(4)                                      # ONE launch, four steps, the neighbours are other processes
    for _ in range(3):
        hs.step(1)
    bad = hs.verify_from_init() + hs.verify_last_step()
    field = torch.cat(comm.all_gather_object(hs.u_tensor().clone()), 0)
    exact = torch.equal(field, reference_steps(initial_field(comm.world, rows, n), 7))
    hs.reset()
    for how in ("memcpy", "nccl"):                  # "nccl" = torch.distributed send/recv: gloo here
        hs.stock_step(how)
    bad += hs.verify_last_step()
    comm.barrier()
    field2 = torch.cat(comm.all_gather_object(hs.u_tensor().clone()), 0)
    exact2 = torch.equal(field2, reference_steps(initial_field(comm.world, rows, n), 2))
    hs.close()
    return {"bad": int(comm.sum(bad)), "exact": exact, "exact_stock": exact2, "leaked": len(emu.live) + len(emu.opened),
            "launches": [l[:3] for l in emu.launches[:4]]}


def _p2p_job(comm, emu, transport):
    """The peer2pear program's Python twin: pairs (2k, 2k+1), unidirectional then bidirectional, verified payload."""
    from hpc_patterns_b200.models.peer2pear import P2PBench

    bench = P2PBench(comm, comm.device, max_bytes=1 << 16, transport=transport, engine="tma", iters=3, label="emu",
                     timeout_s=20.0)
    out = []
    for nbytes in (4096, 1 << 16):
        r = bench.run(nbytes)
        out.append({"bytes": nbytes, "mismatches": r.mismatches, "lines": r.lines(with_size=True),
                    "row": r.row()})
    launches = bench.launches
    bench.close()
    return {"runs": out, "launches": launches, "leaked": len(emu.live) + len(emu.opened)}


def _allreduce_job(comm, emu, algo):
    """The allreduce miniapp's Python twin: VA = rank, VC = 0 -> every element P(P-1)/2, float and int."""
    import contextlib

    from hpc_patterns_b200.models import allreduce as ar

    if algo == "main-a":                                   # the program itself: -a must agree on two-shot (no multicast)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            rc = ar.main(["-a", "-p", "10", "--iters", "2", "--type", "int"])
        return {"rc": rc, "stdout": buf.getvalue(), "leaked": len(emu.live) + len(emu.opened)}
    res = []
    # the stock-library rows go through gloo here, which has no 16-bit integer reduction
    for dtype in ("float", "int", "double") + (() if algo in ("nccl", "ring-nccl") else ("short", "uchar")):
        app = ar.AllreduceMiniapp(comm, comm.device, 10, dtype, algo, timeout_s=20.0)
        with contextlib.redirect_stdout(io.StringIO()) as buf:
            r = app.run(iters=2, warmup=1)
        app.close()
        res.append({"dtype": dtype, "mismatches": r.mismatches, "passed": f"Passed {comm.rank}" in buf.getvalue(),
                    "launches": app.launches})
    return {"results": res, "leaked": len(emu.live) + len(emu.opened)}


def _bench_job(comm_unused, emu, extras):
    import importlib.util

    argv = ["bench.py", "--gpus", "2", "--steps", "4", "--warmup", "3", "--bytes", "65536", "--tile-kb", "1",
            "--preheat-ms", "1", "--blocks", "2", "--e2e-steps", "2"] + ([] if extras else ["--no-extras"])
    sys.argv = argv
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    bench.cpu_concurency = lambda impl: {"impl": impl, "stub": True}
    out, real = io.StringIO(), sys.stdout
    sys.stdout = out
    try:
        rc = bench.main()
    finally:
        sys.stdout = real
    return {"rc": rc, "stdout": out.getvalue()}


def _worker(rank, world, port, job, arg, q):
    try:
        sys.path.insert(0, ROOT)
        os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                          MASTER_PORT=str(port))
        os.environ.pop("HPCP_DEVICE", None)
        import torch.distributed as dist

        dist.init_process_group("gloo", rank=rank, world_size=world)
        from hpc_patterns_b200.parallel.comm import Comm
        from tests.emu_device import SharedEmuNative, TickingEvent, install

        emu = SharedEmuNative()
        install(setattr, emu)
        torch.cuda.Event = TickingEvent
        torch.cuda.is_available = lambda: True
        if job in ("ring", "p2p", "allreduce"):
            comm = Comm()
            res = {"ring": _ring_job, "p2p": _p2p_job, "allreduce": _allreduce_job}[job](comm, emu, arg)
            if not (job == "allreduce" and arg == "main-a"):       # main() closes the Comm it made
                comm.close()
        else:
            res = _bench_job(None, emu, arg)
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok", res))
    except Exception:
        q.put((rank, "error", traceback.format_exc()))


def _run(world, port, job, arg):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, job, arg, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = {}
    try:
        for _ in range(world):
            rank, status, payload = q.get(timeout=150)
            assert status == "ok", f"rank {rank}:\n{payload}"
            results[rank] = payload
    finally:
        for p in procs:
            p.join(timeout=20)
            if p.is_alive():
                p.kill()
    return results


@pytest.mark.parametrize("world,mode,port", [(2, "pull", 29741), (2, "push", 29742), (3, "pull", 29743), (4, "push", 29744)])
def test_ranks_in_separate_processes_step_against_each_other(world, mode, port):
    res = _run(world, port, "ring", mode)
    for rank, r in res.items():
        assert r["bad"] == 0 and r["exact"] and r["exact_stock"], (rank, r)
        assert r["leaked"] == 0
        assert tuple(r["launches"][0]) == (mode, 0, 4), "the first launch ran four steps against live neighbours"


@pytest.mark.parametrize("extras,port", [(False, 29751), (True, 29752)])
def test_bench_line_at_two_ranks(extras, port):
    res = _run(2, port, "bench", extras)
    assert res[0]["rc"] == 0 and res[1]["rc"] == 0
    assert res[1]["stdout"].strip() == "", "only rank 0 prints"
    lines = [l for l in res[0]["stdout"].splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["n_gpus"] == 2 and d["config"]["parallelism"] == "ring2" and d["config"]["global_batch"] == 2
    assert d["wrong_words"] == 0 and d["e2e"]["wrong_words"] == 0
    assert d["value"] == pytest.approx(2 * 2 * 65536 / (d["ms_per_step"] * 1e-3) / 1e9, abs=0.006)
    roof = d["roofline"]
    assert roof["nvlink_ms"] > 0 and roof["bound_ms"] == max(roof["hbm_ms"], roof["nvlink_ms"])
    assert d["frac_of_nvlink_450_nominal"] is not None and d["per_gpu_per_direction_GBps"] > 0
    if extras:
        assert d["stock"]["wrong_words"] == 0
        assert d["stock"]["nccl_sendrecv_ms"] is not None or "nccl_error" in d
        assert d["speedup_vs_stock_memcpy"] > 0 and d["rows_1"]["wrong_words"] == 0


@pytest.mark.parametrize("world,transport,port", [(2, "put", 29761), (2, "get", 29762), (2, "sendrecv", 29763),
                                                  (4, "memcpy", 29764), (2, "nccl", 29765), (4, "hybrid", 29766)])
def test_peer2pear_python_twin(world, transport, port):
    res = _run(world, port, "p2p", transport)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for run in r["runs"]:
            assert run["mismatches"] == 0, (rank, run)
            assert run["row"]["ranks"] == world and run["row"]["transport"] == transport
    lines = res[0]["runs"][1]["lines"]
    assert any("Unidirectional Bandwidth:" in l for l in lines) and any("Bidirectional Bandwidth:" in l for l in lines)
    assert all(r["launches"] > 0 for r in res.values()) or transport == "nccl"


@pytest.mark.parametrize("world,algo,port", [(2, "ring", 29771), (4, "ring", 29772), (4, "ring-unfused", 29773),
                                             (4, "twoshot", 29774), (2, "nccl", 29775), (3, "ring-nccl", 29776)])
def test_allreduce_python_twin(world, algo, port):
    res = _run(world, port, "allreduce", algo)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"], (rank, x)


def test_allreduce_program_dash_a_agrees_on_two_shot():
    res = _run(4, 29781, "allreduce", "main-a")
    assert all(r["rc"] == 0 and r["leaked"] == 0 for r in res.values())
    assert "# -a: twoshot" in res[0]["stdout"] and "# -a:" not in res[1]["stdout"]
    for rank, r in res.items():
        assert f"Passed {rank}" in r["stdout"]
    assert "Elapsed (max over ranks, min of 2)" in res[0]["stdout"]
