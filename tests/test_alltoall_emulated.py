"""The all-to-all's Python layer without a GPU: ``VirtualAlltoall`` and ``ops.alltoall`` on the emulated device of
tests/alltoall_emu.py in one process, and ``AlltoallMiniapp`` in 2-4 ``gloo`` processes through the multi-process
harness of tests/test_multiprocess_emulated.py.  Results are compared byte for byte with recv[r][p] == send[p][r].
The same emulated device with a planted fault in one rank's walk (a misrouted block, a skipped local block, a short
tail) makes ``run()`` report mismatches on exactly the ranks that were hit."""
import contextlib
import io

import numpy as np
import pytest
import torch

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import alltoall as a2a
from hpc_patterns_b200.models.alltoall import AlltoallMiniapp, VirtualAlltoall
from hpc_patterns_b200.ops import alltoall as ops
from hpc_patterns_b200.parallel.local import LocalComm
from tests.alltoall_emu import AlltoallEmuNative, install

_HARNESS_WORKER = mp_harness._worker


def _a2a_job(comm, emu, arg):
    """``run()`` (the miniapp's seeded check), then one all-to-all of random bytes against the torch permutation."""
    algo, _fault, block_bytes = arg
    P = comm.world
    app = AlltoallMiniapp(comm, comm.device, block_bytes, algo, timeout_s=20.0)
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        r = app.run(iters=2, warmup=1)
    own = app.mismatches()
    data = torch.from_numpy(np.random.default_rng(7 + comm.rank).integers(0, 256, (P, block_bytes), dtype=np.uint8))
    app.send.tensor().copy_(data.reshape(-1))
    app.recv.tensor().fill_(0xEE)
    comm.barrier()
    app.pads.device_barrier(0)
    app.run_once()
    comm.barrier()
    want = ops.all_to_all_reference(comm.all_gather_object(data))[comm.rank]
    exact = torch.equal(app.recv.tensor().view(P, block_bytes), want)
    send_kept = torch.equal(app.send.tensor().view(P, block_bytes), data)
    app.close()
    return {"row": r.row(), "own": own, "stdout": buf.getvalue(), "exact": exact, "send_kept": send_kept,
            "leaked": len(emu.live) + len(emu.opened)}


def _a2a_worker(*args):
    """The harness's worker with the all-to-all emulated device (and the job's planted fault), running the job above."""
    from tests.alltoall_emu import use_in_worker

    use_in_worker(args[4][1])
    mp_harness._allreduce_job = _a2a_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,block_bytes,port", [(2, "push", 48, 29961), (3, "pull", 4096 + 16, 29962),
                                                         (4, "push", 16, 29963), (4, "pull", 1040, 29964),
                                                         (3, "nccl", 64, 29965)])
def test_python_twin_in_gloo_processes(world, algo, block_bytes, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _a2a_worker)
    res = mp_harness._run(world, port, "allreduce", (algo, None, block_bytes))
    for rank, r in res.items():
        assert r["leaked"] == 0
        assert r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"] and r["send_kept"], (rank, r)
        assert r["row"] == {"pattern": "alltoall", "variant": algo, "ranks": world, "block_bytes": block_bytes,
                            "ms": 2.0, "GBps_sent_per_rank": pytest.approx((world - 1) * block_bytes / 2e6),
                            "ctas": 0 if algo == "nccl" else 3, "mismatches": 0}


# the ranks whose receive buffer a fault of rank 1's walk (tests/alltoall_emu.py) damages, at 3 ranks
_HIT = {"misroute": {0, 2}, "skip-local": {1}, "short-tail": {0}}


@pytest.mark.parametrize("fault,algo,port", [("misroute", "push", 29971), ("skip-local", "pull", 29972),
                                             ("short-tail", "push", 29973), ("short-tail", "pull", 29974)])
def test_planted_faults_are_reported_on_the_ranks_hit(fault, algo, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _a2a_worker)
    res = mp_harness._run(3, port, "allreduce", (algo, fault, 4096 + 16))
    hit = _HIT[fault] if algo == "push" or fault != "short-tail" else {1}   # pull: rank 1 reads rank 0's block short
    for rank, r in res.items():
        assert r["row"]["mismatches"] > 0, (rank, r)
        if rank in hit:
            assert r["own"] > 0 and f"FAILED {rank}: {r['own']} wrong words" in r["stdout"] and not r["exact"]
        else:
            assert r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"], (rank, r)
    if fault == "short-tail":
        assert sum(r["own"] for r in res.values()) == 4, "one 16-byte vector = 4 words"


@pytest.fixture
def emu(monkeypatch):
    e = AlltoallEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_alltoall_in_one_process(emu, algo, world):
    gen = torch.Generator().manual_seed(world)
    for block_bytes in (16, 48, 4096 + 16):
        v = VirtualAlltoall(world, block_bytes, algo)
        try:
            for launch in range(3):
                sends = [torch.randint(0, 256, (world, block_bytes), dtype=torch.uint8, generator=gen)
                         for _ in range(world)]
                v.load(sends)
                for app in v.ranks:
                    app.recv.tensor().fill_(launch)
                v.run_once()
                out = v.results()
                want = ops.all_to_all_reference(sends)
                assert all(torch.equal(o, w) for o, w in zip(out, want)), (block_bytes, launch)
                assert all(torch.equal(app.send.tensor().view(world, block_bytes), s) for app, s in zip(v.ranks, sends))
            assert [app.pads.ticket_issued for app in v.ranks] == [3 * emu.ctas] * world
            assert [app.pads.barrier_epoch for app in v.ranks] == [3] * world
        finally:
            v.close()


def test_load_views_any_dtype_as_bytes(emu):
    v = VirtualAlltoall(2, 32, "push")
    try:
        sends = [torch.arange(16, dtype=torch.float32) * (r + 1) for r in range(2)]
        v.load(sends)
        v.run_once()
        out = v.results()
        assert torch.equal(out[0][1].view(torch.float32), sends[1][:8])
        assert torch.equal(out[1][0].view(torch.float32), sends[0][8:])
        with pytest.raises(ValueError, match="must hold 2 x 32 bytes"):
            v.load([torch.zeros(48, dtype=torch.uint8)] * 2)
    finally:
        v.close()


def test_a_node_barrier_nobody_arrives_at_is_not_hidden(emu):
    """One process: rank 0 alone cannot complete (its barrier needs rank 1), and the synchronize that observes it says
    so instead of returning a half-finished exchange."""
    v = VirtualAlltoall(2, 16, "push")
    try:
        with torch.cuda.device(0), torch.cuda.stream(v.streams[0]):
            v.ranks[0].run_once()
        with pytest.raises(RuntimeError, match="node barrier 1, rank 1"):
            v.synchronize()
    finally:
        v.close()


def test_refusal_words_are_the_same_in_every_layer(emu):
    C = emu.real
    assert C.all_to_all_refusal(2, 40) == ops.BLOCK_ERROR and C.all_to_all_refusal(2, 0) == ops.BLOCK_ERROR
    assert C.all_to_all_refusal(17, 16) == ops.WORLD_ERROR and C.all_to_all_refusal(0, 16) == ops.WORLD_ERROR
    assert C.all_to_all_refusal(16, 16) == "" and C.ALL_TO_ALL_OVERLAP_ERROR == ops.OVERLAP_ERROR
    for world, block, words in ((2, 40, ops.BLOCK_ERROR), (17, 16, ops.WORLD_ERROR), (2, 0, ops.BLOCK_ERROR)):
        with pytest.raises(ValueError) as e:
            AlltoallMiniapp(LocalComm(0, world), 0, block)
        assert str(e.value) == words
        with pytest.raises(ValueError, match=words):
            ops.all_to_all([0] * world, [0] * world, [0] * world, 0, 0, 0, block, 1)
    with pytest.raises(ValueError, match=ops.BLOCK_ERROR):
        VirtualAlltoall(2, 24)
    buf = emu.alloc(64)
    with pytest.raises(ValueError) as e:
        ops.all_to_all([buf], [buf + 16], [0], 0, 0, 0, 32, 1)
    assert str(e.value) == ops.OVERLAP_ERROR
    with pytest.raises(ValueError, match="algo must be one of"):
        AlltoallMiniapp(LocalComm(0, 2), 0, 16, algo="ring")
    with pytest.raises(ValueError, match="virtual ranks run"):
        VirtualAlltoall(2, 16, "nccl")
    assert a2a.pair_seed(0, 0, 0) != a2a.POISON_SEED
