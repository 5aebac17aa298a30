"""``bin/alltoall --cpu --counts``: the all-to-all-v's host-only run (threads as ranks; the verdict, recv_counts and the
staggered walk of packed segments from the same plan header the kernel uses) at 1-16 ranks and rows of 16 B, 48 B and
4 KiB + 16 B, its report line and JSON row, ``--sweep``, the usage errors before anything is allocated, and the ctest
entries."""
import json
import os
import re
import subprocess

import pytest

from hpc_patterns_b200.models.alltoall import draw_counts, mean_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["pattern", "variant", "ranks", "block_bytes", "ms", "GBps_sent_per_rank", "ctas", "mismatches", "counts",
        "row_bytes", "max_bytes_into_a_rank"]


def _cli(bin_dir, args, cpu=True):
    return subprocess.run([os.path.join(bin_dir, "alltoall")] + (["--cpu"] if cpu else []) + args, cwd=ROOT,
                          capture_output=True, text=True, timeout=300)


@pytest.mark.parametrize("kind", ["random", "skewed"])
@pytest.mark.parametrize("row_bytes", [16, 48, 4096 + 16], ids=["16B", "48B", "4KiB+16B"])
@pytest.mark.parametrize("ranks", [1, 2, 3, 5, 8, 16])
def test_cpu_walk_at_every_rank_count(bin_dir, tmp_path, ranks, row_bytes, kind):
    rows = tmp_path / "rows.jsonl"
    block = 4 * row_bytes
    p = _cli(bin_dir, ["-n", str(ranks), "--counts", kind, "--row-bytes", str(row_bytes), "--block-bytes", str(block),
                       "--iters", "2", "--warmup", "1", "--json", str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    assert sorted(re.findall(r"^Passed (\d+)$", p.stdout, re.M), key=int) == [str(r) for r in range(ranks)]
    assert "FAILED" not in p.stdout
    line = [l for l in p.stdout.splitlines() if l.startswith("Elapsed")]
    assert len(line) == 1 and f"| alltoallv host-alltoallv {kind} P={ranks} B={block} R={row_bytes} host-threads |" in line[0]
    assert line[0].endswith("GB/s sent per rank")
    (row,) = [json.loads(l) for l in rows.read_text().splitlines()]
    assert list(row) == KEYS
    assert row["pattern"] == "alltoallv" and row["variant"] == "host" and row["ranks"] == ranks
    assert row["block_bytes"] == block and row["row_bytes"] == row_bytes and row["counts"] == kind
    assert row["mismatches"] == 0 and row["ctas"] == 0 and row["ms"] > 0
    # the timed iteration is one of the two drawn after the warm-up (iterations 1 and 2); the CLI and the Python twin
    # draw the same matrices
    into = [max(sum(m[p][q] for p in range(ranks)) for q in range(ranks)) * row_bytes
            for m in (draw_counts(kind, ranks, mean_rows(block, row_bytes), it) for it in (1, 2))]
    assert row["max_bytes_into_a_rank"] in into
    if kind == "skewed":
        assert row["max_bytes_into_a_rank"] == 2 * ranks * 4 * row_bytes     # the hot column at the capacity


def test_cpu_sweep_one_row_per_power_of_two(bin_dir, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli(bin_dir, ["-n", "3", "--counts", "random", "--sweep", "--block-bytes", "8192", "--iters", "1", "--json",
                       str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    sizes = [16 << k for k in range(10)]
    got = [json.loads(l) for l in rows.read_text().splitlines()]
    assert [r["block_bytes"] for r in got] == sizes and all(r["mismatches"] == 0 for r in got)
    assert p.stdout.count("Elapsed") == len(sizes) and p.stdout.count("Passed") == 3 * len(sizes)


@pytest.mark.parametrize("args,words", [
    (["--counts", "random", "--row-bytes", "40"], "all-to-all-v: row_bytes must be a positive multiple of 16"),
    (["--counts", "random", "--row-bytes", "0"], "all-to-all-v: row_bytes must be a positive multiple of 16"),
    (["--counts", "skewed", "-n", "17"], "all-to-all: world must be between 1 and 16 ranks"),
    (["--counts", "uniform"], "--counts must be random, skewed or equal"),
    (["--row-bytes", "32"], "--row-bytes needs --counts"),
    (["--counts", "random", "--row-bytes", "1x"], "--row-bytes: not a byte count"),
    (["--counts", "random", "--pull", "--stock", "memcpy"], "--stock memcpy is refused with --pull"),
])
@pytest.mark.parametrize("cpu", [True, False], ids=["cpu", "device"])
def test_usage_errors_before_allocation(bin_dir, args, words, cpu):
    p = _cli(bin_dir, args, cpu=cpu)
    assert p.returncode == 1 and words in p.stderr and "Passed" not in p.stdout, p.stdout + p.stderr
    assert "No devices" not in p.stderr


def test_help(bin_dir):
    p = _cli(bin_dir, ["--help"], cpu=False)
    assert p.returncode == 0 and "--counts K" in p.stdout and "--row-bytes R" in p.stdout


def test_ctest_entries():
    text = open(os.path.join(ROOT, "CMakeLists.txt")).read()
    tests = dict(re.findall(r"add_test\(NAME (all-to-all-v[\w.]*) COMMAND alltoall ([^)]*)\)", text))
    assert set(tests) == {"all-to-all-v", "all-to-all-v.pull", "all-to-all-v.memcpy", "all-to-all-v.host",
                          "all-to-all-v.skewed.host"}
    assert all(tests[n].startswith("-n 4 --counts random") for n in ("all-to-all-v", "all-to-all-v.pull",
                                                                     "all-to-all-v.memcpy"))
    assert "--pull" in tests["all-to-all-v.pull"] and "--stock memcpy" in tests["all-to-all-v.memcpy"]
    assert all("--cpu" in tests[n] for n in ("all-to-all-v.host", "all-to-all-v.skewed.host"))


@pytest.mark.parametrize("name", ["all-to-all-v.host", "all-to-all-v.skewed.host"])
def test_host_ctest_commands_pass(bin_dir, name):
    text = open(os.path.join(ROOT, "CMakeLists.txt")).read()
    args = re.search(rf"add_test\(NAME {re.escape(name)} COMMAND alltoall ([^)]*)\)", text).group(1).split()
    p = subprocess.run([os.path.join(bin_dir, "alltoall")] + args, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "FAILED" not in p.stdout and "Passed 0" in p.stdout, p.stdout + p.stderr
