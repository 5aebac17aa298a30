"""The reduce-scatter's and all-gather's Python layer without a GPU, on the emulated device of
tests/gather_scatter_emu.py: ``ReduceScatterMiniapp`` and ``AllgatherMiniapp`` in 2-4 ``gloo`` processes through the
multi-process harness of tests/test_multiprocess_emulated.py (the constant-data or seeded check of ``run()``, its JSON
row and ``Passed`` on every rank, the ``nccl`` arms, one tensor-level call that must not synchronise the host), the
virtual-rank drivers in one process bit for bit against the references, the refusals before anything is allocated, and
planted faults (a rank that reduces its neighbour's segment, a misplaced block) reported on exactly the ranks hit."""
import contextlib
import io

import numpy as np
import pytest
import torch

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models.allreduce import ReduceScatterMiniapp, VirtualReduceScatter
from hpc_patterns_b200.models.alltoall import AllgatherMiniapp, VirtualAllgather
from hpc_patterns_b200.ops import allreduce as rs_ops
from hpc_patterns_b200.ops import alltoall as ag_ops
from hpc_patterns_b200.parallel.local import LocalComm
from tests.gather_scatter_emu import GatherScatterEmuNative, install
from tests.reduce_scatter_oracle import bits_equal, expected, make_inputs

_HARNESS_WORKER = mp_harness._worker


@contextlib.contextmanager
def _no_host_sync(comm):
    """Any host synchronisation (device, stream or a host barrier with the peers) inside the block raises."""
    def refuse(*a, **k):
        raise AssertionError("the tensor-level call synchronised the host")
    saved = torch.cuda.synchronize, comm.barrier
    torch.cuda.synchronize, comm.barrier = refuse, refuse
    try:
        yield
    finally:
        torch.cuda.synchronize, comm.barrier = saved


def _job(comm, emu, arg):
    kind, algo, dtype, op, size = arg
    P, me = comm.world, comm.rank
    if kind == "rs":
        app = ReduceScatterMiniapp(comm, comm.device, size, dtype, op, algo, timeout_s=20.0)
    else:
        app = AllgatherMiniapp(comm, comm.device, size, algo, timeout_s=20.0)
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        r = app.run(iters=2, warmup=1)
    own = app.mismatches()
    exact = True
    if algo != "nccl":
        rng = np.random.default_rng(11 + me)
        if kind == "rs" and (dtype, op) != ("float", "sum"):
            pass                                    # the tensor-level call is checked on the float sum
        elif kind == "rs":
            x = torch.from_numpy(rng.integers(-1000, 1000, P * app.n).astype(np.float32))
            xs = comm.all_gather_object(x)
            comm.barrier()
            with _no_host_sync(comm):
                out = app.reduce_scatter(x)
            comm.barrier()
            exact = bits_equal(out.clone(), expected(xs, me, "sum", "float"), "float") == 0
        else:
            x = torch.from_numpy(rng.integers(0, 256, size, dtype=np.uint8))
            xs = comm.all_gather_object(x)
            comm.barrier()
            with _no_host_sync(comm):
                out = app.all_gather(x)
            comm.barrier()
            exact = torch.equal(out.clone(), torch.stack(xs))
    app.close()
    return {"row": r.row(), "own": own, "stdout": buf.getvalue(), "exact": exact,
            "leaked": len(emu.live) + len(emu.opened)}


def _worker(*args):
    from tests.gather_scatter_emu import use_in_worker

    use_in_worker(args[4][5] if len(args[4]) > 5 else None)
    mp_harness._allreduce_job = lambda comm, emu, arg: _job(comm, emu, arg[:5])
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,dtype,op,port", [(2, "float", "sum", 29981), (3, "int", "bxor", 29982),
                                                 (4, "float", "sum", 29980),
                                                 (4, "2int", "minloc", 29983), (3, "uchar", "sum", 29984),
                                                 (4, "double", "max", 29985)])
def test_reduce_scatter_twin_in_gloo_processes(world, dtype, op, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _worker)
    res = mp_harness._run(world, port, "allreduce", ("rs", "direct", dtype, op, 8))
    for rank, r in res.items():
        assert r["leaked"] == 0 and r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"], (rank, r)
        row = r["row"]
        assert row["pattern"] == "reduce_scatter" and row["algo"] == "direct" and row["mismatches"] == 0
        assert row["type"] == dtype and row["op"] == op and row["ranks"] == world and row["ms"] == 2.0


@pytest.mark.parametrize("world,algo,block,port", [(2, "push", 48, 29986), (3, "pull", 4096 + 16, 29987),
                                                   (4, "push", 16, 29988)])
def test_allgather_twin_in_gloo_processes(world, algo, block, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _worker)
    res = mp_harness._run(world, port, "allreduce", ("ag", algo, None, None, block))
    for rank, r in res.items():
        assert r["leaked"] == 0 and r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"], (rank, r)
        assert r["row"] == {"pattern": "allgather", "variant": algo, "ranks": world, "block_bytes": block, "ms": 2.0,
                            "GBps_sent_per_rank": pytest.approx((world - 1) * block / 2e6), "ctas": 3,
                            "mismatches": 0}


@pytest.mark.parametrize("kind,port", [("rs", 29989), ("ag", 29990)])
def test_nccl_arms_in_gloo_processes(kind, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _worker)
    arg = ("rs", "nccl", "float", "max", 8) if kind == "rs" else ("ag", "nccl", None, None, 64)
    res = mp_harness._run(2, port, "allreduce", arg)
    for rank, r in res.items():
        assert r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["row"]["mismatches"] == 0, (rank, r)


@pytest.mark.parametrize("kind,fault,hit,port", [("rs", "neighbour-segment", {1}, 29991), ("ag", "misplace", {0}, 29992)])
def test_planted_faults_are_reported_on_the_ranks_hit(kind, fault, hit, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _worker)
    arg = ("rs", "direct", "float", "sum", 8, fault) if kind == "rs" else ("ag", "push", None, None, 64, fault)
    res = mp_harness._run(3, port, "allreduce", arg)
    for rank, r in res.items():
        assert r["row"]["mismatches"] > 0, (rank, r)
        if rank in hit:
            assert r["own"] > 0 and f"FAILED {rank}" in r["stdout"] and not r["exact"], (rank, r)
        else:
            assert r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"], (rank, r)


@pytest.fixture
def emu(monkeypatch):
    e = GatherScatterEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype,op", [("float", "sum"), ("int", "prod"), ("short", "lor"), ("float_int", "maxloc")])
def test_virtual_reduce_scatter_in_one_process(emu, dtype, op, world):
    n = 16 // emu.elem_size(dtype) * 3
    v = VirtualReduceScatter(world, n, dtype, op)
    try:
        for launch in range(3):
            sends = make_inputs(world, n, dtype, op, seed=5, launch=launch)
            v.load([torch.frombuffer(bytearray(s), dtype=torch.uint8) if isinstance(s, bytes) else s for s in sends])
            v.run_once()
            got = v.results()
            for r in range(world):
                g = got[r].numpy().tobytes() if isinstance(sends[0], bytes) else got[r]
                assert bits_equal(g, expected(sends, r, op, dtype), dtype) == 0, (launch, r)
        assert [app.pads.ticket_issued for app in v.ranks] == [3 * emu.ctas] * world
    finally:
        v.close()


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_allgather_in_one_process(emu, algo, world):
    gen = torch.Generator().manual_seed(world)
    v = VirtualAllgather(world, 4096 + 16, algo)
    try:
        for launch in range(3):
            sends = [torch.randint(0, 256, (4096 + 16,), dtype=torch.uint8, generator=gen) for _ in range(world)]
            v.load(sends)
            v.run_once()
            out = v.results()
            assert all(torch.equal(o, ag_ops.all_gather_reference(sends)) for o in out), launch
        assert [app.pads.barrier_epoch for app in v.ranks] == [3] * world
    finally:
        v.close()


def test_refusal_words_are_the_same_in_every_layer(emu):
    C = emu.real
    for world, n, dtype, words in ((2, 3, "float", C.REDUCE_SCATTER_COUNT_ERROR),
                                   (17, 4, "float", C.REDUCE_SCATTER_WORLD_ERROR)):
        assert C.reduce_scatter_refusal(world, n, dtype, "sum") == words
        with pytest.raises(ValueError) as e:
            rs_ops.reduce_scatter([0] * world, 0, [0] * world, 0, 0, 0, n, 1, dtype=dtype)
        assert str(e.value) == words
    for world, block, words in ((2, 40, C.ALL_GATHER_BLOCK_ERROR), (17, 16, C.ALL_GATHER_WORLD_ERROR)):
        assert C.all_gather_refusal(world, block) == words
        with pytest.raises(ValueError) as e:
            AllgatherMiniapp(LocalComm(0, world), 0, block)
        assert str(e.value) == words
    with pytest.raises(ValueError, match="band reduces integer types only"):
        ReduceScatterMiniapp(LocalComm(0, 2), 0, 8, "float", "band")
    buf = emu.alloc(256)
    with pytest.raises(ValueError) as e:
        rs_ops.reduce_scatter([buf, buf + 128], buf + 16, [0, 0], 0, 0, 0, 4, 1)
    assert str(e.value) == C.REDUCE_SCATTER_OVERLAP_ERROR
    with pytest.raises(ValueError) as e:
        ag_ops.all_gather([buf + 16, buf + 128], [buf, buf + 160], [0, 0], 0, 0, 0, 16, 1)
    assert str(e.value) == C.ALL_GATHER_OVERLAP_ERROR
    with pytest.raises(ValueError, match="rank out of range"):
        rs_ops.reduce_scatter([buf, buf + 128], buf + 192, [0, 0], 0, 0, 2, 4, 1)
    with pytest.raises(ValueError, match="rank out of range"):
        ag_ops.all_gather([buf, buf + 128], [buf + 32, buf + 160], [0, 0], 0, 0, -1, 16, 1)
    assert not emu.launches
