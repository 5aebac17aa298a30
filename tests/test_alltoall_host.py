"""``bin/alltoall --cpu``: the all-to-all's host-only plumbing run (threads as ranks, the kernel's staggered walk as
memcpy + a barrier) at 1-16 ranks, its report line and JSON row, the refusals as usage errors before anything is
allocated, the ctest entries, and the Python front door on a box without a GPU."""
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ODD_VECTORS_ABOVE_1MIB = (65536 + 1) * 16


def _cli(bin_dir, args, cpu=True):
    return subprocess.run([os.path.join(bin_dir, "alltoall")] + (["--cpu"] if cpu else []) + args, cwd=ROOT,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("block_bytes", [16, 48, ODD_VECTORS_ABOVE_1MIB], ids=["16B", "48B", "odd-vectors"])
@pytest.mark.parametrize("ranks", [1, 2, 3, 5, 8, 16])
def test_cpu_walk_at_every_rank_count(bin_dir, tmp_path, ranks, block_bytes):
    rows = tmp_path / "rows.jsonl"
    iters = ["--iters", "1", "--warmup", "1"] if block_bytes > 64 else []
    p = _cli(bin_dir, ["-n", str(ranks), "--block-bytes", str(block_bytes), "--json", str(rows)] + iters)
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(re.findall(r"^Passed (\d+)$", p.stdout, re.M), key=int) == [str(r) for r in range(ranks)]
    assert "FAILED" not in p.stdout
    line = [l for l in p.stdout.splitlines() if l.startswith("Elapsed")]
    assert len(line) == 1 and f"| alltoall host-alltoall P={ranks} B={block_bytes} host-threads |" in line[0]
    assert line[0].endswith("GB/s sent per rank")
    (row,) = [json.loads(l) for l in rows.read_text().splitlines()]
    assert list(row) == ["pattern", "variant", "ranks", "block_bytes", "ms", "GBps_sent_per_rank", "ctas", "mismatches"]
    assert row["pattern"] == "alltoall" and row["variant"] == "host" and row["ranks"] == ranks
    assert row["block_bytes"] == block_bytes and row["mismatches"] == 0 and row["ctas"] == 0 and row["ms"] > 0
    assert (row["GBps_sent_per_rank"] > 0) == (ranks > 1)


def test_cpu_sweep_one_row_per_power_of_two(bin_dir, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli(bin_dir, ["-n", "3", "--sweep", "--block-bytes", "8192", "--iters", "1", "--json", str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    sizes = [16 << k for k in range(10)]
    got = [json.loads(l) for l in rows.read_text().splitlines()]
    assert [r["block_bytes"] for r in got] == sizes and all(r["mismatches"] == 0 for r in got)
    assert p.stdout.count("Elapsed") == len(sizes) and p.stdout.count("Passed") == 3 * len(sizes)


@pytest.mark.parametrize("args,words", [
    (["--block-bytes", "40"], "all-to-all: block_bytes must be a positive multiple of 16"),
    (["--block-bytes", "0"], "all-to-all: block_bytes must be a positive multiple of 16"),
    (["--block-bytes", "8"], "all-to-all: block_bytes must be a positive multiple of 16"),
    (["-n", "17"], "all-to-all: world must be between 1 and 16 ranks"),
    (["-n", "0"], "all-to-all: world must be between 1 and 16 ranks"),
    (["--pull", "--stock", "memcpy"], "--stock memcpy is refused with --pull"),
    (["--stock", "nccl"], "--stock must be memcpy"),
    (["--block-bytes", "1x"], "--block-bytes: not a byte count"),
])
@pytest.mark.parametrize("cpu", [True, False], ids=["cpu", "device"])
def test_refusals_are_usage_errors_before_allocation(bin_dir, args, words, cpu):
    """With or without --cpu the words come before anything else: on a GPU-less box the device path would otherwise
    say "No devices"; on a GPU box nothing has been allocated yet."""
    p = _cli(bin_dir, args, cpu=cpu)
    assert p.returncode == 1 and words in p.stderr and "Passed" not in p.stdout, p.stdout + p.stderr
    assert "No devices" not in p.stderr


def test_help(bin_dir):
    p = _cli(bin_dir, ["--help"], cpu=False)
    assert p.returncode == 0 and "--stock memcpy" in p.stdout and "--block-bytes B" in p.stdout


def test_ctest_entries():
    """The GPU cases run 4 ranks like the allreduce's; the host cases (the ones ctest -R host runs anywhere) pass."""
    text = open(os.path.join(ROOT, "CMakeLists.txt")).read()
    tests = dict(re.findall(r"add_test\(NAME (alltoall[\w.]*) COMMAND alltoall ([^)]*)\)", text))
    assert set(tests) == {"alltoall", "alltoall.pull", "alltoall.memcpy", "alltoall.host", "alltoall.sweep.host"}
    assert all(tests[n].startswith("-n 4") for n in ("alltoall", "alltoall.pull", "alltoall.memcpy"))
    assert "--pull" in tests["alltoall.pull"] and "--stock memcpy" in tests["alltoall.memcpy"]
    assert "add_executable(alltoall csrc/miniapps/alltoall.cu)" in text
    assert "bin/alltoall" in open(os.path.join(ROOT, "Makefile")).read()


@pytest.mark.parametrize("name", ["alltoall.host", "alltoall.sweep.host"])
def test_host_ctest_commands_pass(bin_dir, name):
    text = open(os.path.join(ROOT, "CMakeLists.txt")).read()
    args = re.search(rf"add_test\(NAME {re.escape(name)} COMMAND alltoall ([^)]*)\)", text).group(1).split()
    p = subprocess.run([os.path.join(bin_dir, "alltoall")] + args, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "FAILED" not in p.stdout and "Passed 0" in p.stdout, p.stdout + p.stderr


def test_front_door_without_gpu(gpu_count):
    if gpu_count:
        pytest.skip("the box has a GPU")
    p = subprocess.run([sys.executable, "-m", "hpc_patterns_b200", "alltoall"], cwd=ROOT, capture_output=True,
                       text=True, timeout=300)
    assert p.returncode == 1 and "Traceback" not in p.stderr
    assert p.stderr.strip() == ("Error: alltoall: no CUDA device (this program runs sm_90a kernels; bin/alltoall --cpu "
                                "is the host-only plumbing run)")
