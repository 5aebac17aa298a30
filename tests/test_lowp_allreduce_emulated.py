"""The allreduce miniapp's Python twin for bfloat16 / half on the emulated device (tests/emu_device.py,
tests/lowp_emu.py): the dtype plumbing of ``AllreduceMiniapp`` / ``VirtualAllreduce`` / ``ops.allreduce``, the ``-a``
choice, and every algorithm as 2 and 3 ``gloo`` processes (harness of tests/test_multiprocess_emulated.py) -- with the
miniapp's own constant-data check and with the oracle's data, bit for bit (tests/lowp_allreduce_oracle.py)."""
import pytest
import torch

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import allreduce as ar
from tests.emu_device import install
from tests.lowp_allreduce_oracle import (LOWP, TORCH_DTYPE, make_inputs, mismatches, ring_expected, rsag_expected,
                                         two_shot_expected)
from tests.lowp_emu import LowpEmuNative

_HARNESS_WORKER = mp_harness._worker


def _expected(algo, vas, rank):
    return (two_shot_expected(vas) if algo == "twoshot" else rsag_expected(vas) if algo == "ring-rsag"
            else ring_expected(vas, rank))


def _lowp_job(comm, emu, algo):
    """Per 16-bit type: ``run()`` (VA = rank, the miniapp's check), then one allreduce of the oracle's data."""
    import contextlib
    import io

    res = []
    for dtype in LOWP:
        app = ar.AllreduceMiniapp(comm, comm.device, 10, dtype, algo, timeout_s=20.0)
        with contextlib.redirect_stdout(io.StringIO()) as buf:
            r = app.run(iters=2, warmup=1)
        vas = make_inputs(comm.world, app.n, dtype, seed=77)
        td = TORCH_DTYPE[dtype]
        app.va.tensor(td).copy_(vas[comm.rank])
        app.vc.tensor(td).zero_()
        comm.barrier()
        app.pads.device_barrier(0)
        app.run_once()
        comm.barrier()
        bad = mismatches(app.vc.tensor(td).clone(), _expected(algo, vas, comm.rank))
        app.close()
        res.append({"dtype": dtype, "mismatches": r.mismatches, "passed": f"Passed {comm.rank}" in buf.getvalue(),
                    "oracle_mismatches": bad, "row_type": r.row()["type"]})
    return {"results": res, "leaked": len(emu.live) + len(emu.opened)}


def _lowp_worker(*args):
    """The harness's worker, with the emulated device that also runs 16-bit ring-rsag, running the job above."""
    from tests.lowp_emu import use_in_worker

    use_in_worker()
    mp_harness._allreduce_job = _lowp_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,port", [(2, "ring", 29801), (3, "ring", 29802), (3, "ring-unfused", 29803),
                                             (2, "twoshot", 29804), (3, "twoshot", 29805), (2, "ring-rsag", 29806),
                                             (3, "ring-rsag", 29807)])
def test_python_twin_in_gloo_processes(world, algo, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _lowp_worker)
    res = mp_harness._run(world, port, "allreduce", algo)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"] and x["oracle_mismatches"] == 0, (rank, x)
            assert x["row_type"] == x["dtype"]


@pytest.fixture
def emu(monkeypatch):
    e = LowpEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("algo", ar.VIRTUAL_ALGOS)
@pytest.mark.parametrize("dtype", LOWP)
def test_virtual_allreduce_in_one_process(emu, dtype, algo):
    """One rank in one process: the whole path (buffers, pads, run_once, results) for the 16-bit types."""
    n = 8 * 1001
    v = ar.VirtualAllreduce(1, n, dtype, algo)
    try:
        for seed in range(2):
            vas = make_inputs(1, n, dtype, seed=seed, kind="subnormal" if seed else "full")
            v.load(vas)
            v.run_once()
            assert mismatches(v.results()[0], _expected(algo, vas, 0)) == 0
    finally:
        v.close()


def test_emulated_device_two_shot_and_ring_are_the_oracles(emu):
    """The emulated kernels themselves, rank by rank, on pointers: what the twins above rely on."""
    world, n = 3, 8 * 3 * 40
    for dtype in LOWP:
        td = TORCH_DTYPE[dtype]
        vas = make_inputs(world, n, dtype, seed=5)
        va = [emu.alloc(2 * n) for _ in range(world)]
        vc = [emu.alloc(2 * n) for _ in range(world)]
        pads = [emu.alloc(4 * 4096) for _ in range(world)]
        for r in range(world):
            emu._arr(va[r], n, dtype)[:] = vas[r]
        for r in range(world):
            emu._arr(vc[r], n, dtype)[r * n // world:(r + 1) * n // world] = 0
        for p in pads:                       # every rank's barrier word already there: the one-thread driver cannot wait
            for r in range(world):
                emu.signal(p + 4 * (emu.real.PAD_BARRIER + r), 1, 0)
        for r in range(world):
            emu.allreduce_two_shot(va, vc, pads, 0, 0, r, n, 1, 0, 0, dtype, 0, 0, 0)
        want = two_shot_expected(vas)
        for r in range(world):
            assert mismatches(emu._arr(vc[r], n, dtype).clone(), want) == 0
        acc = emu._arr(vc[0], n, dtype)
        acc.zero_()
        emu.accumulate(va[1], vc[0], n, dtype, 0)
        emu.accumulate(va[2], vc[0], n, dtype, 0)
        assert mismatches(acc.clone(), (torch.zeros(n, dtype=td) + vas[1]) + vas[2]) == 0


def test_dash_a_and_tensor_ops_take_the_16bit_types(monkeypatch):
    from hpc_patterns_b200.ops import allreduce as ops

    class C:
        def multicast_supported(self, device):
            return True

    class World8:
        world = 8

        def min(self, x):
            raise AssertionError("decided locally")

    monkeypatch.setattr(ar, "native", lambda: C())
    for dtype in LOWP:
        algo, why = ar.choose_collective(World8(), 0, dtype, 25)
        assert algo == "twoshot" and "fp32" in why
    assert ops.dtype_name(torch.empty(1, dtype=torch.bfloat16)) == "bfloat16"
    assert ops.dtype_name(torch.empty(1, dtype=torch.float16)) == "half"
    with pytest.raises(TypeError):
        ops.dtype_name(torch.empty(1, dtype=torch.float64))
    assert ar._TORCH_DTYPE["bfloat16"] is torch.bfloat16 and ar._TORCH_DTYPE["half"] is torch.float16
