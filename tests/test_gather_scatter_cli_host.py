"""``bin/reduce_scatter --cpu`` and ``bin/allgather --cpu`` (program names of the allreduce and alltoall miniapps): the
host-only plumbing runs at several rank counts, types and ops, their report lines and JSON rows, the options each
program refuses as usage errors before anything is allocated, and the ctest entries, whose host commands pass."""
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cli(bin_dir, prog, args):
    return subprocess.run([os.path.join(bin_dir, prog)] + args, cwd=ROOT, capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("ranks", [1, 3, 4, 16])
@pytest.mark.parametrize("dtype,op", [("float", "sum"), ("uchar", "sum"), ("bfloat16", "sum"), ("half", "prod"),
                                      ("int", "bxor"), ("ushort", "lor"), ("double", "min"), ("short_int", "maxloc")])
def test_reduce_scatter_cpu(bin_dir, tmp_path, ranks, dtype, op):
    rows = tmp_path / "rows.jsonl"
    p = _cli(bin_dir, "reduce_scatter", ["--cpu", "-n", str(ranks), "-p", "10", "--type", dtype, "--op", op,
                                         "--iters", "2", "--json", str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(re.findall(r"^Passed (\d+)$", p.stdout, re.M), key=int) == [str(r) for r in range(ranks)]
    row = json.loads(rows.read_text())
    assert row["pattern"] == "reduce_scatter" and row["algo"] == "host" and row["mismatches"] == 0
    assert row["type"] == dtype and row["op"] == op and row["ranks"] == ranks
    assert f"reduce_scatter host {dtype} P={ranks}" in p.stdout


@pytest.mark.parametrize("ranks", [1, 4, 5])
@pytest.mark.parametrize("block", [16, 48, 4096 + 16])
def test_allgather_cpu(bin_dir, tmp_path, ranks, block):
    rows = tmp_path / "rows.jsonl"
    p = _cli(bin_dir, "allgather", ["--cpu", "-n", str(ranks), "--block-bytes", str(block), "--json", str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(re.findall(r"^Passed (\d+)$", p.stdout, re.M), key=int) == [str(r) for r in range(ranks)]
    row = json.loads(rows.read_text())
    assert row == {"pattern": "allgather", "variant": "host", "ranks": ranks, "block_bytes": block, "ms": row["ms"],
                   "GBps_sent_per_rank": row["GBps_sent_per_rank"], "ctas": 0, "mismatches": 0}


@pytest.mark.parametrize("args,words", [(["-a"], "reduce_scatter: -a is an allreduce option"),
                                        (["--algo", "ring"], "reduce_scatter: --algo"),
                                        (["--coll", "twoshot"], "reduce_scatter: --coll"),
                                        (["--slots", "2"], "reduce_scatter: --slots"),
                                        (["--pull"], "reduce_scatter: --pull"),
                                        (["-H"], "reduce_scatter: -H"), (["-S"], "reduce_scatter: -S"),
                                        (["-R"], "reduce_scatter: -R"),
                                        (["--type", "float", "--op", "band"], "band reduces integer types only"),
                                        (["-n", "17"], "reduce-scatter: world must be between 1 and 16 ranks")])
@pytest.mark.parametrize("cpu", [True, False])
def test_reduce_scatter_usage_errors(bin_dir, args, words, cpu):
    p = _cli(bin_dir, "reduce_scatter", (["--cpu"] if cpu else []) + args)
    assert p.returncode == 1 and words in p.stderr and "Passed" not in p.stdout, p.stdout + p.stderr


@pytest.mark.parametrize("args,words", [(["--counts", "random"], "allgather: --counts and --row-bytes"),
                                        (["--block-bytes", "24"], "all-gather: block_bytes must be a positive"),
                                        (["-n", "17"], "all-gather: world must be between 1 and 16 ranks"),
                                        (["--stock", "memcpy", "--pull"], "--stock memcpy is refused with --pull")])
@pytest.mark.parametrize("cpu", [True, False])
def test_allgather_usage_errors(bin_dir, args, words, cpu):
    p = _cli(bin_dir, "allgather", (["--cpu"] if cpu else []) + args)
    assert p.returncode == 1 and words in p.stderr and "Passed" not in p.stdout, p.stdout + p.stderr


def _ctests():
    text = open(os.path.join(ROOT, "CMakeLists.txt")).read()
    out = {}
    for name, cmd in re.findall(r"add_test\(NAME ((?:reduce_scatter|allgather)[\w.]*)\s+COMMAND ([^)]*)\)", text):
        prog = "reduce_scatter" if "{rs}" in cmd or "/reduce_scatter" in cmd else "allgather"
        out[name] = (prog, cmd.split()[1:])
    return out


def test_ctest_entries():
    t = _ctests()
    gpu = {n for n in t if not n.endswith(".host")}
    assert gpu == {"allgather", "allgather.pull", "allgather.memcpy", "reduce_scatter", "reduce_scatter.bfloat16"}
    assert all(t[n][1][:2] == ["-n", "4"] for n in gpu)
    host = {n for n in t if n.endswith(".host")}
    assert {t[n][1][t[n][1].index("-n") + 1] for n in host if t[n][0] == "reduce_scatter"} >= {"1", "3", "4"}
    assert {t[n][1][t[n][1].index("-n") + 1] for n in host if t[n][0] == "allgather"} == {"1", "4", "5"}
    make = open(os.path.join(ROOT, "Makefile")).read()
    assert "ln -sf allreduce bin/reduce_scatter" in make and "ln -sf alltoall bin/allgather" in make


@pytest.mark.parametrize("name", sorted(n for n in _ctests() if n.endswith(".host")))
def test_host_ctest_commands_pass(bin_dir, name):
    prog, args = _ctests()[name]
    p = _cli(bin_dir, prog, args)
    assert p.returncode == 0 and "FAILED" not in p.stdout and "Passed 0" in p.stdout, p.stdout + p.stderr
