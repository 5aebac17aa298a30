"""prod / min / max through the allreduce miniapp's Python twin on the emulated device (tests/op_emu.py), and through
``bin/allreduce --cpu``: the ``op`` plumbing of ``AllreduceMiniapp`` / ``VirtualAllreduce``, the ``-a`` choice, the
argument errors, every algorithm as 2 and 3 ``gloo`` processes (harness of tests/test_multiprocess_emulated.py) with
the miniapp's own constant-data check and with the oracle's data bit for bit (tests/reduce_op_oracle.py), and sum
output that keeps its shape."""
import json
import os
import subprocess

import pytest

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import allreduce as ar
from tests.emu_device import install
from tests.op_emu import OpEmuNative
from tests.reduce_op_oracle import (OPS, TORCH_DTYPE, TYPES, kinds, make_inputs, mismatches, ring_expected,
                                    rsag_expected, two_shot_expected)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HARNESS_WORKER = mp_harness._worker
_MP_TYPES = ("float", "uint", "short", "bfloat16")


def _expected(algo, vas, rank, op, dtype):
    return (two_shot_expected(vas, op, dtype) if algo == "twoshot" else rsag_expected(vas, op, dtype)
            if algo == "ring-rsag" else ring_expected(vas, rank, op, dtype))


def _ops_job(comm, emu, algo):
    """Per op and type: ``run()`` (the miniapp's constant-data check), then one allreduce of the oracle's data."""
    import contextlib
    import io

    res = []
    for op in OPS:
        for dtype in _MP_TYPES if algo != "nccl" else ("float", "int"):
            app = ar.AllreduceMiniapp(comm, comm.device, 10, dtype, algo, timeout_s=20.0, op=op)
            with contextlib.redirect_stdout(io.StringIO()) as buf:
                r = app.run(iters=2, warmup=1)
            bad = 0
            if algo != "nccl":
                vas = make_inputs(comm.world, app.n, dtype, seed=77, op=op, kind=kinds(op, dtype)[-1])
                td = TORCH_DTYPE[dtype]
                app.va.tensor(td).copy_(vas[comm.rank])
                app.vc.tensor().fill_(0xFF)
                comm.barrier()
                app.pads.device_barrier(0)
                app.run_once()
                comm.barrier()
                bad = mismatches(app.vc.tensor(td).clone(), _expected(algo, vas, comm.rank, op, dtype))
            app.close()
            res.append({"op": op, "dtype": dtype, "mismatches": r.mismatches, "oracle_mismatches": bad,
                        "passed": f"Passed {comm.rank}" in buf.getvalue(), "row_op": r.row().get("op")})
    return {"results": res, "leaked": len(emu.live) + len(emu.opened)}


def _ops_worker(*args):
    """The harness's worker with the op-aware emulated device, running the job above."""
    from tests.op_emu import use_in_worker

    use_in_worker()
    mp_harness._allreduce_job = _ops_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,port", [(2, "ring", 29851), (3, "ring", 29852), (3, "ring-unfused", 29853),
                                             (2, "twoshot", 29854), (3, "twoshot", 29855), (3, "ring-rsag", 29856),
                                             (2, "nccl", 29857)])
def test_python_twin_ops_in_gloo_processes(world, algo, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _ops_worker)
    res = mp_harness._run(world, port, "allreduce", algo)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"] and x["oracle_mismatches"] == 0, (rank, x)
            assert x["row_op"] == x["op"]


@pytest.fixture
def emu(monkeypatch):
    e = OpEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("algo", ar.VIRTUAL_ALGOS)
@pytest.mark.parametrize("op", OPS)
def test_virtual_allreduce_in_one_process(emu, op, algo):
    """One rank: VC must come out as VA whatever it held (the ops overwrite it)."""
    for dtype in ("double", "ushort", "half"):
        n = 8 * 1001
        v = ar.VirtualAllreduce(1, n, dtype, algo, op=op)
        try:
            vas = make_inputs(1, n, dtype, seed=3, op=op, kind=kinds(op, dtype)[0])
            v.load(vas)
            for app in v.ranks:
                app.vc.tensor().fill_(0xFF)
            v.run_once()
            assert mismatches(v.results()[0], _expected(algo, vas, 0, op, dtype)) == 0
        finally:
            v.close()


def test_sum_rows_keep_their_shape():
    row = ar.AllreduceResult("ring", "float", 4, 1024, 1.0, 0, 4).row()
    assert "op" not in row
    assert ar.AllreduceResult("ring", "float", 4, 1024, 1.0, 0, 4, "max").row()["op"] == "max"


def test_choose_collective_with_op(monkeypatch):
    class C:
        def multicast_supported(self, device):
            return True

    class World8:
        world = 8

        def min(self, x):
            return x

    monkeypatch.setattr(ar, "native", lambda: C())
    assert ar.choose_collective(World8(), 0, "float", 25)[0] == "nvls"
    assert ar.choose_collective(World8(), 0, "float", 25, op="sum")[0] == "nvls"
    for op in ("max", "min", "prod", "product"):
        algo, why = ar.choose_collective(World8(), 0, "float", 25, op)
        assert algo == "twoshot" and "sums only" in why


def test_argument_errors(emu):
    comm = None                 # every refusal comes before the communicator is used
    with pytest.raises(ValueError, match="nvls"):
        ar.AllreduceMiniapp(comm, 0, 10, "float", "nvls", op="max")
    for algo in ("nccl", "ring-nccl"):
        for dtype in ("uint", "ulong", "ushort"):
            for op in ("min", "max"):
                with pytest.raises(ValueError, match="signed"):
                    ar.AllreduceMiniapp(comm, 0, 10, dtype, algo, op=op)
    with pytest.raises(ValueError, match="op must be"):
        ar.AllreduceMiniapp(comm, 0, 10, "float", "ring", op="avg")
    with pytest.raises(ValueError, match="op must be"):
        ar.VirtualAllreduce(1, 1024, "float", "ring", op="bxor")
    assert ar.reduce_op("product") == "prod"
    assert [ar.expected_value(6, op) for op in ("sum", "max", "min", "prod")] == [15, 5, 1, 8]
    assert ar.expected_value(16, "prod") == 16


# ------------------------------------------------------------ bin/allreduce --cpu ----
def _cli(bin_dir, args):
    return subprocess.run([os.path.join(bin_dir, "allreduce"), "--cpu"] + args, cwd=ROOT, capture_output=True,
                          text=True, timeout=120)


@pytest.mark.parametrize("algo", [["--algo", "ring"], ["--algo", "ring-unfused"], ["--algo", "ring-rsag"], ["-a"]],
                         ids=["ring", "ring-unfused", "ring-rsag", "a"])
@pytest.mark.parametrize("op", OPS)
def test_cli_cpu_every_type(bin_dir, op, algo):
    for t in TYPES:
        for n in ("3", "16"):
            p = _cli(bin_dir, ["-n", n, "-p", "8", "--type", t, "--op", op] + algo)
            assert p.returncode == 0 and p.stdout.count("Passed") == int(n), (t, n, p.stdout + p.stderr)
            assert f"op={op}" in p.stdout


def test_cli_cpu_refusals_and_rows(bin_dir, tmp_path):
    p = _cli(bin_dir, ["-n", "4", "-a", "--coll", "nvls", "--op", "max"])
    assert p.returncode != 0 and "sum-only" in p.stderr
    p = _cli(bin_dir, ["-n", "4", "--op", "avg"])
    assert p.returncode != 0 and "unknown --op" in p.stderr
    rows = tmp_path / "rows.jsonl"
    for extra in ([], ["--op", "sum"], ["--op", "product"]):
        p = _cli(bin_dir, ["-n", "3", "-p", "6", "--json", str(rows)] + extra)
        assert p.returncode == 0, p.stdout + p.stderr
    sum_row, sum_row2, prod_row = [json.loads(x) for x in rows.read_text().splitlines()]
    assert "op" not in sum_row and "op" not in sum_row2 and prod_row["op"] == "prod"
    assert "op=" not in _cli(bin_dir, ["-n", "3", "-p", "6"]).stdout
