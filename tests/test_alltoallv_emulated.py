"""The all-to-all-v's Python layer without a GPU: ``VirtualAlltoallv``, ``AlltoallvMiniapp`` and ``ops.alltoall`` on the
emulated device of tests/alltoallv_emu.py (which runs the bound plan rules) in one process, and ``AlltoallvMiniapp`` in
2-4 ``gloo`` processes through the multi-process harness of tests/test_multiprocess_emulated.py.  Faults planted in one
rank's launch are reported by the miniapp's own check on exactly the ranks whose receive buffer or recv_counts they
damage, a refused matrix moves nothing, and the refusal and verdict words are the same in every layer."""
import contextlib
import io

import pytest
import torch

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import alltoall as a2a
from hpc_patterns_b200.models.alltoall import AlltoallvMiniapp, VirtualAlltoallv
from hpc_patterns_b200.ops import alltoall as ops
from hpc_patterns_b200.parallel.local import LocalComm
from tests.alltoallv_emu import FAULTS, AlltoallvEmuNative, install

_HARNESS_WORKER = mp_harness._worker


def _a2av_job(comm, emu, arg):
    """``run()`` (the miniapp's seeded check), then one exchange of random rows against the torch reference."""
    algo, kind, row_bytes = arg
    P, mean = comm.world, 3
    app = AlltoallvMiniapp(comm, comm.device, row_bytes, 2 * P * mean, algo, timeout_s=20.0)
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        r = app.run(kind, mean * row_bytes, iters=2, warmup=1)
    own = app.mismatches()
    gen = torch.Generator().manual_seed(11 + comm.rank)
    splits = torch.randint(0, 2 * mean + 1, (P,), generator=gen)
    x = torch.randint(0, 256, (int(splits.sum()), row_bytes), dtype=torch.uint8, generator=gen)
    comm.barrier()
    rows, rc = app.exchange(x, splits)
    app.check()
    comm.barrier()
    counts = comm.all_gather_object(splits.tolist())
    want = ops.all_to_all_v_reference(comm.all_gather_object(x), counts, row_bytes)[comm.rank]
    exact = torch.equal(rows[: want.shape[0]], want) and rc.tolist() == [counts[p][comm.rank] for p in range(P)]
    app.close()
    return {"row": r.row(), "own": own, "stdout": buf.getvalue(), "exact": exact,
            "leaked": len(emu.live) + len(emu.opened)}


def _a2av_worker(*args):
    from tests.alltoallv_emu import use_in_worker

    use_in_worker(None)
    mp_harness._allreduce_job = _a2av_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,kind,row_bytes,port", [(2, "push", "random", 48, 29981),
                                                            (3, "pull", "skewed", 4096 + 16, 29982),
                                                            (4, "push", "skewed", 16, 29983),
                                                            (3, "nccl", "random", 32, 29984)])
def test_python_twin_in_gloo_processes(world, algo, kind, row_bytes, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _a2av_worker)
    res = mp_harness._run(world, port, "allreduce", (algo, kind, row_bytes))
    for rank, r in res.items():
        assert r["leaked"] == 0
        assert r["own"] == 0 and f"Passed {rank}" in r["stdout"] and r["exact"], (rank, r)
        row = r["row"]
        assert row["pattern"] == "alltoallv" and row["variant"] == algo and row["ranks"] == world
        assert row["mismatches"] == 0 and row["counts"] == kind and row["row_bytes"] == row_bytes
        assert row["ctas"] == (0 if algo == "nccl" else 3) and row["max_bytes_into_a_rank"] > 0


@pytest.fixture
def emu(monkeypatch):
    e = AlltoallvEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_alltoallv_in_one_process(emu, algo, world):
    gen = torch.Generator().manual_seed(world)
    for row_bytes in (16, 48, 4096 + 16):
        cap = 2 * world * 4
        v = VirtualAlltoallv(world, row_bytes, cap, algo)
        try:
            for launch in range(3):
                m = a2a.draw_counts(("random", "skewed", "equal")[launch], world, 4, launch)
                sends = [torch.randint(0, 256, (cap, row_bytes), dtype=torch.uint8, generator=gen) for _ in range(world)]
                v.load(sends, m)
                for app in v.ranks:
                    app.recv.tensor().fill_(launch)
                v.run_once()
                out = v.results()
                want = ops.all_to_all_v_reference(sends, m, row_bytes)
                for r, ((rows, rc), w) in enumerate(zip(out, want)):
                    assert torch.equal(rows, w) and rc.tolist() == [m[p][r] for p in range(world)]
                    assert bool((v.ranks[r].recv.tensor()[w.numel():] == launch).all())
                assert v.verdicts() == [0] * world
            assert [app.pads.ticket_issued for app in v.ranks] == [3 * emu.ctas] * world
            assert [app.pads.barrier_epoch for app in v.ranks] == [3] * world
        finally:
            v.close()


@pytest.mark.parametrize("fault", ["inclusive-prefix", "short-segment", "no-recv-counts", "row-recv-offset"])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_planted_faults_are_reported_on_the_ranks_hit(emu, fault, algo):
    """The miniapp's seeded check (``initialize`` / ``mismatches``) on drawn count matrices: a rank reports wrong words
    exactly when its receive buffer or recv_counts differ from what a fault-free launch leaves there."""
    world, mean, R = 3, 4, 48
    emu.fault, emu.fault_rank = fault, 1
    v = VirtualAlltoallv(world, R, 2 * world * mean, algo)
    ever = set()
    try:
        for it in range(6):
            for app in v.ranks:
                app.initialize("random", mean)
            m = v.ranks[0].matrix
            sends = [app.send.tensor().clone() for app in v.ranks]
            expect = [app.recv.tensor().clone() for app in v.ranks]
            for r, w in enumerate(ops.all_to_all_v_reference(sends, m, R)):
                expect[r][: w.numel()] = w.reshape(-1)
            v.run_once()
            v.synchronize()
            hit = {r for r, app in enumerate(v.ranks)
                   if not torch.equal(app.recv.tensor(), expect[r]) or app.recv_counts.tolist() != [m[p][r] for p in range(world)]}
            bad = {r for r, app in enumerate(v.ranks) if app.mismatches() > 0}
            assert bad == hit, (it, m, bad, hit)
            if fault == "no-recv-counts" or algo == "pull":
                assert hit <= {1}
            ever |= hit
        assert ever, "the fault never hit a rank"
    finally:
        v.close()


@pytest.mark.parametrize("algo", ["push", "pull"])
@pytest.mark.parametrize("rule", [1, 2, 3])
def test_a_refused_matrix_moves_nothing_and_a_faulty_copy_is_seen(emu, algo, rule):
    world, cap = 3, 10
    m = [[2, 2, 2] for _ in range(world)]
    if rule == 1:
        m[2][0] = -1
    elif rule == 2:
        m[1] = [4, 4, 4]
    else:
        m[0][2] = m[1][2] = m[2][2] = 4
    gen = torch.Generator().manual_seed(rule)
    for fault in (None, "copy-refused"):
        emu.fault, emu.fault_rank = fault, 1
        v = VirtualAlltoallv(world, 32, cap, algo)
        try:
            sends = [torch.randint(0, 256, (cap, 32), dtype=torch.uint8, generator=gen) for _ in range(world)]
            v.load(sends, m)
            for app in v.ranks:
                app.recv.tensor().fill_(0xC3)
            v.run_once()
            assert v.verdicts() == [rule] * world
            with pytest.raises(ValueError) as e:
                v.results()
            assert str(e.value) == ops.VERDICT_WORDS[rule] == emu.real.all_to_all_v_verdict_words(rule)
            changed = {r for r, app in enumerate(v.ranks) if not bool((app.recv.tensor() == 0xC3).all())}
            if fault is None:
                assert changed == set()
            else:
                assert changed == ({1} if algo == "pull" else {q for q in range(world) if m[1][q] > 0} - set()), changed
            assert [app.recv_counts.tolist() for app in v.ranks] == [[m[p][r] for p in range(world)] for r in range(world)]
        finally:
            v.close()


def test_exchange_refusals_and_check(emu):
    """``exchange`` itself runs in the gloo processes above (one process cannot hold a rank's barrier open while its
    peers enqueue); here: its shape refusals, and ``check()`` raising the verdict's words once synchronised."""
    v = VirtualAlltoallv(2, 16, 8, "push")
    try:
        with pytest.raises(ValueError, match="send capacity is 8"):
            v.ranks[0].exchange(torch.zeros(9, 4), torch.tensor([1, 2]))
        with pytest.raises(ValueError, match="must hold 16 bytes"):
            v.ranks[0].exchange(torch.zeros(2, 8), torch.tensor([1, 2]))
        v.load([torch.zeros(2, 16, dtype=torch.uint8)] * 2, [[-1, 0], [1, 1]])
        v.run_once()
        v.synchronize()
        for app in v.ranks:
            with pytest.raises(ValueError, match=ops.VERDICT_WORDS[1]):
                app.check()
    finally:
        v.close()


def test_refusal_words_are_the_same_in_every_layer(emu):
    C = emu.real
    assert C.all_to_all_v_refusal(2, 40, 1, 1) == ops.ROW_ERROR and C.all_to_all_v_refusal(2, 0, 1, 1) == ops.ROW_ERROR
    assert C.all_to_all_v_refusal(17, 16, 1, 1) == ops.WORLD_ERROR and C.all_to_all_v_refusal(0, 16, 1, 1) == ops.WORLD_ERROR
    assert C.all_to_all_v_refusal(2, 16, 0, 1) == ops.CAPACITY_ERROR == C.all_to_all_v_refusal(2, 16, 1, -1)
    assert C.all_to_all_v_refusal(16, 16, 1, 1) == "" and C.ALL_TO_ALL_V_COUNTS_OVERLAP_ERROR == ops.COUNTS_OVERLAP_ERROR
    for k in (1, 2, 3):
        assert C.all_to_all_v_verdict_words(k) == ops.VERDICT_WORDS[k]
    assert C.all_to_all_v_verdict_words(0) == "" and C.ALLTOALLV_ACCEPTED == 0
    assert (C.ALLTOALLV_NEGATIVE, C.ALLTOALLV_SEND_CAPACITY, C.ALLTOALLV_RECV_CAPACITY) == (1, 2, 3)
    for world, rb, cap, words in ((2, 40, 4, ops.ROW_ERROR), (17, 16, 4, ops.WORLD_ERROR), (2, 16, 0, ops.CAPACITY_ERROR)):
        with pytest.raises(ValueError) as e:
            AlltoallvMiniapp(LocalComm(0, world), 0, rb, cap)
        assert str(e.value) == words
        with pytest.raises(ValueError, match=words):
            ops.all_to_all_v([0] * world, [0] * world, [0] * world, 0, 0, [0] * world, 0, 0, 0, rb, cap, cap, 1)
    buf = emu.alloc(256)
    with pytest.raises(ValueError) as e:
        ops.all_to_all_v([buf], [buf + 16], [buf + 128], buf + 192, 0, [0], 0, 0, 0, 16, 2, 2, 1)
    assert str(e.value) == ops.OVERLAP_ERROR
    with pytest.raises(ValueError) as e:
        ops.all_to_all_v([buf], [buf + 64], [buf + 128], buf + 132, 0, [0], 0, 0, 0, 16, 2, 2, 1)
    assert str(e.value) == ops.COUNTS_OVERLAP_ERROR
    with pytest.raises(ValueError, match="algo must be one of"):
        AlltoallvMiniapp(LocalComm(0, 2), 0, 16, 4, algo="ring")
    with pytest.raises(ValueError, match="virtual ranks run"):
        VirtualAlltoallv(2, 16, 4, "nccl")
    with pytest.raises(ValueError, match="random, skewed or equal"):
        a2a.draw_counts("uniform", 2, 1, 0)
    assert set(FAULTS) == {"inclusive-prefix", "row-recv-offset", "copy-refused", "no-recv-counts", "short-segment",
                           "rows-below-8"}
