"""band / bor / bxor / land / lor / lxor through the allreduce miniapp's Python twin on the emulated device
(tests/bitop_emu.py), and through ``bin/allreduce --cpu``: every algorithm as 2 and 3 ``gloo`` processes (harness of
tests/test_multiprocess_emulated.py) with the miniapp's own constant-data check and with tests/bitop_oracle.py's data
bit for bit, one rank in one process, every op x integer type x algorithm of the CLI at 1, 3 and 16 ranks, and the
refusals: floating types everywhere, ``nccl``, ``nvls``."""
import json
import os
import subprocess

import pytest

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import allreduce as ar
from tests.bitop_emu import BitOpEmuNative
from tests.bitop_oracle import (BIT_OPS, FLOAT_TYPES, INT_TYPES, KINDS, TORCH_DTYPE, allreduce_expected, make_inputs,
                                mismatches)
from tests.emu_device import install

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HARNESS_WORKER = mp_harness._worker
_MP_TYPES = ("int", "ushort", "uchar", "ulong")


def _bitops_job(comm, emu, algo):
    """Per op and type: ``run()`` (the miniapp's constant-data check), then one allreduce of the oracle's data (not for
    ring-nccl, whose buffers are torch tensors the oracle step does not reach)."""
    import contextlib
    import io

    res = []
    for i, op in enumerate(BIT_OPS):
        for dtype in _MP_TYPES:
            app = ar.AllreduceMiniapp(comm, comm.device, 10, dtype, algo, timeout_s=20.0, op=op)
            with contextlib.redirect_stdout(io.StringIO()) as buf:
                r = app.run(iters=2, warmup=1)
            bad = 0
            if algo != "ring-nccl":
                vas = make_inputs(comm.world, app.n, dtype, seed=31 + i, kind=KINDS[i % len(KINDS)])
                app.va.tensor(TORCH_DTYPE[dtype]).copy_(vas[comm.rank])
                app.vc.tensor().fill_(0xFF)
                comm.barrier()
                app.pads.device_barrier(0)
                app.run_once()
                comm.barrier()
                bad = mismatches(app.vc.tensor(TORCH_DTYPE[dtype]).clone(), allreduce_expected(vas, op, dtype))
            app.close()
            res.append({"op": op, "dtype": dtype, "mismatches": r.mismatches, "oracle_mismatches": bad,
                        "passed": f"Passed {comm.rank}" in buf.getvalue(), "row_op": r.row().get("op")})
    return {"results": res, "leaked": len(emu.live) + len(emu.opened)}


def _bitops_worker(*args):
    """The harness's worker with the bit-op-aware emulated device, running the job above."""
    from tests.bitop_emu import use_in_worker

    use_in_worker()
    mp_harness._allreduce_job = _bitops_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,port", [(2, "ring", 29871), (3, "ring", 29872), (3, "ring-unfused", 29873),
                                             (2, "twoshot", 29874), (3, "twoshot", 29875), (3, "ring-rsag", 29876),
                                             (2, "ring-nccl", 29877)])
def test_python_twin_bitops_in_gloo_processes(world, algo, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _bitops_worker)
    res = mp_harness._run(world, port, "allreduce", algo)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"] and x["oracle_mismatches"] == 0, (rank, x)
            assert x["row_op"] == x["op"]


@pytest.fixture
def emu(monkeypatch):
    e = BitOpEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("algo", ar.VIRTUAL_ALGOS)
@pytest.mark.parametrize("op", BIT_OPS)
def test_virtual_allreduce_in_one_process(emu, op, algo):
    """One rank: VC must come out as VA, unnormalised, whatever it held (the ops overwrite it)."""
    for dtype in ("long", "ushort", "uchar"):
        n = 16 * 1001
        v = ar.VirtualAllreduce(1, n, dtype, algo, op=op)
        try:
            vas = make_inputs(1, n, dtype, seed=3, kind="high")
            v.load(vas)
            for app in v.ranks:
                app.vc.tensor().fill_(0xFF)
            v.run_once()
            assert mismatches(v.results()[0], vas[0]) == 0
        finally:
            v.close()


def test_argument_errors(emu):
    comm = None                 # every refusal comes before the communicator is used
    for op in BIT_OPS:
        for dtype in FLOAT_TYPES:
            for algo in ("ring", "twoshot", "ring-nccl"):
                with pytest.raises(ValueError, match="op must be .*integer types only"):
                    ar.AllreduceMiniapp(comm, 0, 10, dtype, algo, op=op)
            with pytest.raises(ValueError, match="op must be"):
                ar.VirtualAllreduce(1, 1024, dtype, "ring", op=op)
        with pytest.raises(ValueError, match="nccl has no"):
            ar.AllreduceMiniapp(comm, 0, 10, "int", "nccl", op=op)
        with pytest.raises(ValueError, match="nvls"):
            ar.AllreduceMiniapp(comm, 0, 10, "int", "nvls", op=op)
        with pytest.raises(ValueError, match="integer types only"):
            ar.main(["--type", "half", "--op", op])
        with pytest.raises(RuntimeError, match=f"for float: {op} reduces integer types only"):
            emu.accumulate(0, 0, 0, "float", 0, op=op)
    assert ar.reduce_op("lxor") == "lxor"
    with pytest.raises(ValueError, match="op must be"):
        ar.reduce_op("bnot")


def test_choose_collective_with_bitops(monkeypatch):
    class C:
        def multicast_supported(self, device):
            return True

    class World8:
        world = 8

        def min(self, x):
            return x

    monkeypatch.setattr(ar, "native", lambda: C())
    for op in BIT_OPS:
        algo, why = ar.choose_collective(World8(), 0, "int", 25, op)
        assert algo == "twoshot" and "sums only" in why


def test_rows_carry_the_op():
    assert ar.AllreduceResult("twoshot", "uchar", 4, 1024, 1.0, 0, 1, "bxor").row()["op"] == "bxor"


# ------------------------------------------------------------ bin/allreduce --cpu ----
def _cli(bin_dir, args, name="allreduce"):
    return subprocess.run([os.path.join(bin_dir, name), "--cpu"] + args, cwd=ROOT, capture_output=True, text=True,
                          timeout=120)


@pytest.mark.parametrize("algo", [["--algo", "ring"], ["--algo", "ring-unfused"], ["--algo", "ring-rsag"], ["-a"]],
                         ids=["ring", "ring-unfused", "ring-rsag", "a"])
@pytest.mark.parametrize("op", BIT_OPS)
def test_cli_cpu_every_integer_type(bin_dir, op, algo):
    for t in INT_TYPES:
        for n in ("1", "3", "16"):
            p = _cli(bin_dir, ["-n", n, "-p", "8", "--type", t, "--op", op] + algo)
            assert p.returncode == 0 and p.stdout.count("Passed") == int(n), (t, n, p.stdout + p.stderr)
            assert f"op={op}" in p.stdout


def test_cli_cpu_typed_binary_and_rows(bin_dir, tmp_path):
    rows = tmp_path / "rows.jsonl"
    for name, op in (("allreduce.int", "land"), ("allreduce.uchar", "bxor"), ("allreduce.long", "bor")):
        p = _cli(bin_dir, ["-n", "5", "-p", "8", "--op", op, "--json", str(rows)], name=name)
        assert p.returncode == 0 and p.stdout.count("Passed") == 5, p.stdout + p.stderr
    got = [json.loads(x) for x in rows.read_text().splitlines()]
    assert [(r["type"], r["op"], r["mismatches"]) for r in got] == [("int", "land", 0), ("uchar", "bxor", 0),
                                                                     ("long", "bor", 0)]


def test_cli_cpu_refusals(bin_dir):
    for args in (["--type", "float", "--op", "band"], ["--op", "lxor"], ["--type", "half", "--op", "lor", "-a"],
                 ["--type", "double", "--op", "bxor", "--algo", "ring-rsag"]):
        p = _cli(bin_dir, ["-n", "3", "-p", "6"] + args)
        assert p.returncode != 0 and "integer types only" in p.stderr and "Passed" not in p.stdout, args
    p = _cli(bin_dir, ["-n", "4", "--type", "int", "-a", "--coll", "nvls", "--op", "band"])
    assert p.returncode != 0 and "sum-only" in p.stderr
    p = _cli(bin_dir, ["-n", "4", "--op", "bnot"])
    assert p.returncode != 0 and "unknown --op" in p.stderr and "lxor" in p.stderr
