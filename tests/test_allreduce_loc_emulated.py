"""maxloc / minloc without a GPU: the allreduce miniapp's Python twin on the emulated device (tests/loc_emu.py) as 1-3
``gloo`` processes for every algorithm (ring-nccl included) and in one process, ``main()`` with a pair type,
``bin/allreduce --cpu`` for every op x pair type x algorithm, the refusals in every layer with their exact words, and
``pack_loc`` / ``unpack_loc`` against ``ctypes`` structs."""
import ctypes
import json
import os
import subprocess

import pytest
import torch

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import allreduce as ar
from hpc_patterns_b200.models.allreduce import (AllreduceMiniapp, VirtualAllreduce, check_op_type, loc_expected,
                                                loc_input)
from hpc_patterns_b200.ops.allreduce import loc_combine, pack_loc, unpack_loc
from tests.emu_device import install
from tests.loc_emu import LocEmuNative
from tests.loc_oracle import (KINDS, LOC_OPS, PAIR_TYPES, allreduce_expected, const_expected, const_input, make_inputs,
                              mismatches, pair_bytes)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HARNESS_WORKER = mp_harness._worker


def _loc_job(comm, emu, algo):
    """``main()`` with a pair type and no --op (the default op is maxloc), or per op and pair type: ``run()`` (the
    miniapp's constant-data check), then one allreduce of the oracle's data, garbage padding and all, from an all-ones
    VC."""
    import contextlib
    import io

    if algo == "main-a":
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            rc = ar.main(["-a", "-p", "8", "--iters", "2", "--type", "double_int"])
        return {"rc": rc, "stdout": buf.getvalue(), "leaked": len(emu.live) + len(emu.opened)}
    res = []
    for i, op in enumerate(LOC_OPS):
        for j, dtype in enumerate(PAIR_TYPES):
            app = ar.AllreduceMiniapp(comm, comm.device, 8, dtype, algo, timeout_s=20.0, op=op)
            with contextlib.redirect_stdout(io.StringIO()) as buf:
                r = app.run(iters=2, warmup=1)
            vas = make_inputs(comm.world, app.n, dtype, seed=41 + 7 * i + j, kind=KINDS[(i + j) % len(KINDS)])
            app.va.tensor(torch.uint8).copy_(torch.frombuffer(bytearray(vas[comm.rank]), dtype=torch.uint8))
            app.vc.tensor(torch.uint8).fill_(0xFF)
            comm.barrier()
            app.pads.device_barrier(0)
            app.run_once()
            comm.barrier()
            bad = mismatches(app.vc.tensor(torch.uint8).numpy().tobytes(), allreduce_expected(op, vas, dtype), dtype)
            app.close()
            res.append({"op": op, "dtype": dtype, "mismatches": r.mismatches, "oracle_mismatches": bad,
                        "passed": f"Passed {comm.rank}" in buf.getvalue(), "row": r.row()})
    return {"results": res, "leaked": len(emu.live) + len(emu.opened)}


def _loc_worker(*args):
    """The harness's worker with the loc-aware emulated device, running the job above."""
    from tests.loc_emu import use_in_worker

    use_in_worker()
    mp_harness._allreduce_job = _loc_job
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world,algo,port", [(2, "ring", 29881), (3, "ring", 29882), (3, "ring-unfused", 29883),
                                             (2, "twoshot", 29884), (3, "twoshot", 29885), (3, "ring-rsag", 29886),
                                             (1, "ring-nccl", 29887), (2, "ring-nccl", 29888), (3, "ring-nccl", 29889)])
def test_python_twin_loc_in_gloo_processes(world, algo, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _loc_worker)
    res = mp_harness._run(world, port, "allreduce", algo)
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"] and x["oracle_mismatches"] == 0, (rank, x)
            assert x["row"]["op"] == x["op"] and x["row"]["type"] == x["dtype"]


def test_main_with_a_pair_type_defaults_to_maxloc(monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _loc_worker)
    res = mp_harness._run(2, 29890, "allreduce", "main-a")
    for rank, r in res.items():
        assert r["rc"] == 0 and r["leaked"] == 0 and f"Passed {rank}" in r["stdout"], r
    assert "twoshot double_int" in res[0]["stdout"] and "op=maxloc" in res[0]["stdout"]


@pytest.fixture
def emu(monkeypatch):
    e = LocEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("algo", ar.VIRTUAL_ALGOS)
@pytest.mark.parametrize("op", LOC_OPS)
def test_virtual_allreduce_in_one_process(emu, op, algo):
    """One rank: VC must come out as a byte copy of VA (garbage padding, NaN payloads), whatever it held; load() and
    results() take and give (values, indices)."""
    for dtype in PAIR_TYPES:
        n = 2 * 1001
        v = ar.VirtualAllreduce(1, n, dtype, algo, op=op)
        try:
            va = make_inputs(1, n, dtype, seed=3, kind="special")[0]
            v.load([unpack_loc(torch.frombuffer(bytearray(va), dtype=torch.uint8), dtype)])
            v.ranks[0].va.tensor(torch.uint8).copy_(torch.frombuffer(bytearray(va), dtype=torch.uint8))
            v.ranks[0].vc.tensor(torch.uint8).fill_(0xFF)
            v.run_once()
            assert v.ranks[0].vc.tensor(torch.uint8).numpy().tobytes() == va
            vals, idx = v.results()[0]
            want_v, want_i = unpack_loc(torch.frombuffer(bytearray(va), dtype=torch.uint8), dtype)
            assert torch.equal(idx, want_i) and torch.equal(vals.view(torch.uint8), want_v.view(torch.uint8))
        finally:
            v.close()


def test_emulated_refusals_use_the_native_words(emu):
    with pytest.raises(RuntimeError, match="op must be maxloc or minloc for 2int: sum reduces arithmetic types only"):
        emu.accumulate(0, 0, 0, "2int", 0)
    with pytest.raises(RuntimeError, match="for int: maxloc reduces value-index pair types only"):
        emu.accumulate(0, 0, 0, "int", 0, op="maxloc")
    with pytest.raises(ValueError, match="op must be maxloc or minloc for float_int: max reduces arithmetic"):
        ar.main(["--type", "float_int", "--op", "max"])


def _cli(bin_dir, args, name="allreduce"):
    return subprocess.run([os.path.join(bin_dir, name), "--cpu"] + args, cwd=ROOT, capture_output=True, text=True,
                          timeout=120)


@pytest.mark.parametrize("algo", [["--algo", "ring"], ["--algo", "ring-unfused"], ["--algo", "ring-rsag"], ["-a"]],
                         ids=["ring", "ring-unfused", "ring-rsag", "a"])
@pytest.mark.parametrize("op", LOC_OPS)
def test_cli_cpu_every_pair_type(bin_dir, op, algo):
    for t in PAIR_TYPES:
        for n in ("1", "3", "16"):
            p = _cli(bin_dir, ["-n", n, "-p", "7", "--type", t, "--op", op] + algo)
            assert p.returncode == 0 and p.stdout.count("Passed") == int(n), (t, n, p.stdout + p.stderr)


def test_cli_cpu_typed_binary_defaults_to_maxloc(bin_dir, tmp_path):
    rows = tmp_path / "rows.jsonl"
    for t in PAIR_TYPES:
        p = _cli(bin_dir, ["-n", "5", "-p", "8", "--json", str(rows)], name="allreduce." + t)
        assert p.returncode == 0 and "op=maxloc" in p.stdout, p.stdout + p.stderr
    got = [json.loads(line) for line in rows.read_text().splitlines()]
    assert [(r["type"], r["op"], r["mismatches"]) for r in got] == [(t, "maxloc", 0) for t in PAIR_TYPES]


@pytest.mark.parametrize("args,words", [
    (["--type", "float_int", "--op", "sum"], "op must be maxloc or minloc for float_int: sum reduces arithmetic types only"),
    (["--type", "short_int", "--op", "band"], "op must be maxloc or minloc for short_int: band reduces arithmetic types only"),
    (["--op", "maxloc"], "op must be sum, prod, min or max for float: maxloc reduces value-index pair types only"),
    (["--type", "long", "--op", "minloc"], "op must be sum, prod, min, max, band, bor, bxor, land, lor or lxor for long: "
                                           "minloc reduces value-index pair types only"),
    (["--type", "double", "--op", "bor"], "op must be sum, prod, min or max for double: bor reduces integer types only"),
    (["--type", "2int", "-a", "--coll", "nvls"], "--coll nvls is sum-only: --op maxloc needs --coll twoshot or auto"),
])
def test_cli_cpu_refusals(bin_dir, args, words):
    p = _cli(bin_dir, ["-n", "3", "-p", "6"] + args)
    assert p.returncode != 0 and words in p.stderr and "Passed" not in p.stdout, p.stderr


@pytest.mark.parametrize("dtype,op,words", [
    ("float_int", "sum", "op must be maxloc or minloc for float_int: sum reduces arithmetic types only"),
    ("float", "maxloc", "op must be sum, prod, min or max for float: maxloc reduces value-index pair types only"),
    ("uchar", "minloc", "op must be sum, prod, min, max, band, bor, bxor, land, lor or lxor for uchar: minloc reduces "
                        "value-index pair types only"),
    ("half", "band", "op must be sum, prod, min or max for half: band reduces integer types only"),
])
def test_python_refusals_use_the_native_words(dtype, op, words):
    with pytest.raises(ValueError) as e:
        check_op_type(op, dtype)
    assert str(e.value) == words
    with pytest.raises(ValueError, match=words):
        VirtualAllreduce(2, 64, dtype, "ring", op=op)
    with pytest.raises(ValueError, match=words):
        AllreduceMiniapp(None, 0, dtype=dtype, op=op)


def test_python_nccl_refuses_loc_ops():
    with pytest.raises(ValueError, match="nccl has no maxloc or minloc"):
        AllreduceMiniapp(None, 0, dtype="float_int", algo="nccl", op="maxloc")


class _FloatInt(ctypes.Structure):
    _fields_ = [("value", ctypes.c_float), ("index", ctypes.c_int)]


class _DoubleInt(ctypes.Structure):
    _fields_ = [("value", ctypes.c_double), ("index", ctypes.c_int)]


class _LongInt(ctypes.Structure):
    _fields_ = [("value", ctypes.c_long), ("index", ctypes.c_int)]


class _TwoInt(ctypes.Structure):
    _fields_ = [("value", ctypes.c_int), ("index", ctypes.c_int)]


class _ShortInt(ctypes.Structure):
    _fields_ = [("value", ctypes.c_short), ("index", ctypes.c_int)]


CSTRUCT = {"float_int": (_FloatInt, torch.float32), "double_int": (_DoubleInt, torch.float64),
           "long_int": (_LongInt, torch.int64), "2int": (_TwoInt, torch.int32), "short_int": (_ShortInt, torch.int16)}


@pytest.mark.parametrize("dtype", PAIR_TYPES)
def test_pack_loc_is_the_c_struct(dtype):
    S, vt = CSTRUCT[dtype]
    assert ctypes.sizeof(S) == pair_bytes(dtype)
    values = torch.tensor([-3, 0, 7, 1000], dtype=vt)
    indices = torch.tensor([2 ** 31 - 1, -2 ** 31, -1, 5], dtype=torch.int32)
    arr = (S * 4)()
    ctypes.memset(arr, 0, ctypes.sizeof(arr))
    for k in range(4):
        arr[k].value, arr[k].index = values[k].item(), int(indices[k])
    buf = pack_loc(values, indices)
    assert buf.dtype == torch.uint8 and bytes(buf.numpy()) == bytes(arr)
    v, i = unpack_loc(buf, dtype)
    assert torch.equal(v, values) and torch.equal(i, indices)


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_ring_nccl_combine_is_the_oracle(op, dtype):
    """loc_combine (ring-nccl's torch combine) folds to the oracle's bytes on every input kind."""
    for kind in KINDS:
        vas = make_inputs(4, 256, dtype, seed=5, kind=kind)
        acc = torch.frombuffer(bytearray(vas[0]), dtype=torch.uint8)
        for v in vas[1:]:
            acc = loc_combine(acc, torch.frombuffer(bytearray(v), dtype=torch.uint8), dtype, op)
        assert bytes(acc.numpy()) == allreduce_expected(op, vas, dtype), kind


@pytest.mark.parametrize("op", LOC_OPS)
def test_model_constant_data_is_the_oracle_table(op):
    for world in range(1, 17):
        assert loc_expected(op, world) == const_expected(op, world)
        assert all(loc_input(op, r, world) == const_input(op, r, world) for r in range(world))
