"""The all-gather kernels (launch_all_gather) on one H100 with virtual ranks: push and pull at 1-8 ranks, blocks from
one 16-byte vector to 64 MiB, random bytes compared bit for bit with torch.cat of every rank's block, three
consecutive launches on the same buffers with fresh data (tickets and epochs carried across launches), the send
blocks unchanged after every launch; the refusals, and the tensor-level call that enqueues without a host sync."""
import json
import os
import subprocess

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from hpc_patterns_b200.models.alltoall import VirtualAllgather
from hpc_patterns_b200.ops.alltoall import all_gather, all_gather_reference

pytestmark = pytest.mark.gpu

_C = hpc_patterns_b200.native()
GATHER_BLOCK_ERROR, GATHER_WORLD_ERROR = _C.ALL_GATHER_BLOCK_ERROR, _C.ALL_GATHER_WORLD_ERROR

BLOCKS = [16, 48, 4096 + 16, 1 << 20, 64 << 20]
LAUNCHES = 3


@pytest.fixture(scope="module", autouse=True)
def first_launches(native):
    """Launch each kernel once on a single rank before the virtual ranks start (as tests/test_gpu_alltoall.py)."""
    for algo in ("push", "pull"):
        v = VirtualAllgather(1, 16, algo)
        v.run_once()
        v.synchronize()
        v.close()


@pytest.mark.parametrize("block_bytes", BLOCKS, ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_ranks_bit_for_bit(algo, world, block_bytes):
    v = VirtualAllgather(world, block_bytes, algo)
    try:
        gen = torch.Generator(device="cuda").manual_seed(1000 * world + block_bytes % 997)
        for launch in range(LAUNCHES):
            sends = [torch.randint(0, 256, (block_bytes,), dtype=torch.uint8, device="cuda", generator=gen)
                     for _ in range(world)]
            v.load(sends)
            for app in v.ranks:
                app.recv.tensor().fill_(0xA5 ^ launch)
            torch.cuda.synchronize()
            v.run_once()
            v.synchronize()
            want = torch.cat([s.reshape(1, -1) for s in sends])
            for r, app in enumerate(v.ranks):
                got = app.recv.tensor().view(world, block_bytes)
                assert torch.equal(got, want), (launch, r, int((got != want).any(dim=1).sum()))
                assert torch.equal(app.send.tensor(), sends[r]), ("send written", launch, r)
            assert [app.pads.ticket_issued for app in v.ranks] == [(launch + 1) * v.ranks[0].launch_ctas] * world
        if block_bytes == 48:
            got = v.results()
            assert torch.equal(got[0], all_gather_reference([s.cpu() for s in sends]))
    finally:
        v.close()


def test_refusals(native):
    with pytest.raises(ValueError, match=GATHER_BLOCK_ERROR):
        VirtualAllgather(2, 24)
    with pytest.raises(ValueError, match="world <= 8"):
        VirtualAllgather(9, 16)
    assert native.all_gather_refusal(17, 16) == GATHER_WORLD_ERROR
    assert native.all_gather_refusal(4, 0) == GATHER_BLOCK_ERROR
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    with pytest.raises(ValueError, match="rank out of range"):
        all_gather([p + 16, p + 1024], [p + 2048, p + 3072], [p, p], 0, 0, -1, 16, 1)
    with pytest.raises(ValueError, match="in-place"):     # my send block inside my receive buffer (MPI_IN_PLACE)
        all_gather([p + 16, p + 1024], [p, p + 2048], [p, p], 0, 0, 0, 16, 1)
    with pytest.raises(Exception, match="in-place"):
        native.all_gather([p + 16, p + 1024], [p, p + 2048], [p, p], 0, 0, 0, 16, 1)
    with pytest.raises(ValueError, match=GATHER_WORLD_ERROR):
        all_gather([p] * 17, [p] * 17, [p] * 17, 0, 0, 0, 16, 1)


@pytest.mark.parametrize("algo", ["push", "pull"])
def test_tensor_level_call_enqueues_without_host_sync(algo):
    world = 4
    v = VirtualAllgather(world, 4096 * 4, algo)
    try:
        for launch in range(2):
            xs = [torch.randn(64, 64, device="cuda") for _ in range(world)]
            torch.cuda.synchronize()
            outs = []
            torch.cuda.set_sync_debug_mode("error")   # any host synchronisation inside the calls raises
            try:
                for app, st, x in zip(v.ranks, v.streams, xs):
                    with torch.cuda.stream(st):
                        outs.append(app.all_gather(x))
            finally:
                torch.cuda.set_sync_debug_mode(0)
            v.synchronize()
            want = torch.stack(xs)
            assert all(o.shape == (world, 64, 64) and torch.equal(o, want) for o in outs), launch
    finally:
        v.close()


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cli(bin_dir, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "allgather"), "-n", "4", "--json", str(rows)] + args, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    got = [json.loads(line) for line in rows.read_text().splitlines()] if rows.exists() else []
    return p, got


@pytest.mark.parametrize("args,variant", [([], "push"), (["--pull"], "pull"), (["--stock", "memcpy"], "memcpy")])
def test_cli_four_ranks(bin_dir, tmp_path, args, variant):
    p, rows = _cli(bin_dir, args + ["--block-bytes", str((4 << 20) + 16), "--iters", "3"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    for r in range(4):
        assert f"Passed {r}" in p.stdout, p.stdout
    assert len(rows) == 1 and rows[0]["pattern"] == "allgather" and rows[0]["variant"] == variant
    assert rows[0]["mismatches"] == 0 and rows[0]["ms"] > 0 and rows[0]["block_bytes"] == (4 << 20) + 16


def test_cli_short_sweep(bin_dir, tmp_path):
    p, rows = _cli(bin_dir, ["--sweep", "--block-bytes", str(1 << 20), "--iters", "2", "--pull"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    sizes = [16 << k for k in range(17)]
    assert [r["block_bytes"] for r in rows] == sizes and all(r["mismatches"] == 0 for r in rows)
    assert p.stdout.count("Passed") == 4 * len(sizes) and "FAILED" not in p.stdout
