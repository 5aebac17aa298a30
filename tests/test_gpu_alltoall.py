"""The all-to-all kernels on one H100 with virtual ranks: push and pull at 1-8 ranks, block sizes from one 16-byte
vector to 64 MiB, random bytes compared bit for bit with the torch permutation recv[r][p] = send[p][r], several
consecutive launches on the same buffers with fresh data (epochs and tickets carried across launches), the send
buffers unchanged after every launch; and bin/alltoall on 4 ranks (push, pull, the stock memcpy shape, a short sweep)."""
import json
import os
import subprocess

import pytest
import torch

from hpc_patterns_b200.models.alltoall import VirtualAlltoall
from hpc_patterns_b200.ops.alltoall import all_to_all_reference

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCKS = [16, 48, 4096 + 16, 1 << 20, 64 << 20]
LAUNCHES = 3


@pytest.fixture(scope="module", autouse=True)
def first_launches(native):
    """Launch each kernel once on a single rank before the virtual ranks start: a process's first launch of a kernel
    can wait for the device to go idle, which a peer's spinning barrier never lets happen."""
    for algo in ("push", "pull"):
        v = VirtualAlltoall(1, 16, algo)
        v.run_once()
        v.synchronize()
        v.close()


@pytest.mark.parametrize("block_bytes", BLOCKS, ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_ranks_bit_for_bit(algo, world, block_bytes):
    v = VirtualAlltoall(world, block_bytes, algo)
    try:
        gen = torch.Generator(device="cuda").manual_seed(1000 * world + block_bytes % 997)
        for launch in range(LAUNCHES):
            sends = [torch.randint(0, 256, (world, block_bytes), dtype=torch.uint8, device="cuda", generator=gen)
                     for _ in range(world)]
            v.load(sends)
            for app in v.ranks:      # poison: a block that is never written cannot pass as last launch's
                app.recv.tensor().fill_(0xA5 ^ launch)
            torch.cuda.synchronize()
            v.run_once()
            v.synchronize()
            want = all_to_all_reference(sends)
            for r, app in enumerate(v.ranks):
                got = app.recv.tensor().view(world, block_bytes)
                assert torch.equal(got, want[r]), (launch, r, int((got != want[r]).any(dim=1).sum()))
                assert torch.equal(app.send.tensor().view(world, block_bytes), sends[r]), ("send written", launch, r)
            assert [app.pads.ticket_issued for app in v.ranks] == [(launch + 1) * v.ranks[0].launch_ctas] * world
        if world > 1 and block_bytes == 48:
            got = v.results()
            assert len(got) == world and got[0].shape == (world, block_bytes) and got[0].device.type == "cpu"
    finally:
        v.close()


def test_load_takes_any_dtype_as_bytes():
    v = VirtualAlltoall(2, 64, "pull")
    try:
        sends = [torch.arange(32, dtype=torch.float32, device="cuda") + 100 * r for r in range(2)]
        v.load(sends)
        v.run_once()
        out = v.results()
        want = all_to_all_reference([s.cpu() for s in sends])
        assert all(torch.equal(o, w) for o, w in zip(out, want))
        assert torch.equal(out[1][0].view(torch.float32), sends[0][16:].cpu())
    finally:
        v.close()


def _cli(bin_dir, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "alltoall"), "-n", "4", "--json", str(rows)] + args, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    got = [json.loads(line) for line in rows.read_text().splitlines()] if rows.exists() else []
    return p, got


@pytest.mark.parametrize("args,variant", [([], "push"), (["--pull"], "pull"), (["--stock", "memcpy"], "memcpy")])
def test_cli_four_ranks(bin_dir, tmp_path, args, variant):
    p, rows = _cli(bin_dir, args + ["--block-bytes", str((4 << 20) + 16), "--iters", "3"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    for r in range(4):
        assert f"Passed {r}" in p.stdout, p.stdout
    assert len(rows) == 1 and rows[0]["variant"] == variant and rows[0]["mismatches"] == 0 and rows[0]["ms"] > 0
    assert rows[0]["ranks"] == 4 and rows[0]["block_bytes"] == (4 << 20) + 16


def test_cli_short_sweep(bin_dir, tmp_path):
    p, rows = _cli(bin_dir, ["--sweep", "--block-bytes", str(1 << 20), "--iters", "2"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    sizes = [16 << k for k in range(17)]
    assert [r["block_bytes"] for r in rows] == sizes and all(r["mismatches"] == 0 for r in rows)
    assert p.stdout.count("Passed") == 4 * len(sizes) and "FAILED" not in p.stdout
