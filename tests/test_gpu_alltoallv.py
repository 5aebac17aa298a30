"""The all-to-all-v kernels on one H100 with virtual ranks: push and pull at 1-8 ranks with rows of 16 B, 48 B and
4 KiB + 16 B, count matrices from random-with-zeros to a column exactly at the receive capacity and a 64 MiB exchange,
three consecutive launches with new counts and bytes, bit for bit against ``all_to_all_v_reference``: the poison past
every total intact, send buffers and counts unchanged, recv_counts exact, tickets and epochs advancing.  The v kernel at
equal counts equals the equal-block kernel; refused count matrices (declared capacities below what is allocated) move
no byte anywhere, every rank reports the same verdict and the next valid launch is exact; ``exchange()`` never
synchronises the host; and bin/alltoall --counts on 4 ranks."""
import json
import os
import subprocess

import pytest
import torch

from hpc_patterns_b200.models.alltoall import VirtualAlltoall, VirtualAlltoallv
from hpc_patterns_b200.ops.alltoall import VERDICT_WORDS, all_to_all_v_reference
from tests.alltoallv_oracle import PATTERNS, counts_for

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = [16, 48, 4096 + 16]
MEAN = 24                       # mean rows per pair; every instance has capacities of 2 * P * MEAN rows


@pytest.fixture(scope="module", autouse=True)
def first_launches(native):
    """Launch each kernel once on a single rank before the virtual ranks start (see test_gpu_alltoall.py)."""
    for algo in ("push", "pull"):
        v = VirtualAlltoallv(1, 16, 4, algo)
        v.load([torch.zeros(4, 16, dtype=torch.uint8, device="cuda")], [[4]])
        v.run_once()
        v.synchronize()
        v.close()


def run_and_check(v, m, gen, launch):
    """Load fresh bytes and `m`, poison every receive buffer, launch, and check everything the test promises."""
    P, R, cap = v.world, v.row_bytes, v.capacity_rows
    sends = [torch.randint(0, 256, (cap, R), dtype=torch.uint8, device="cuda", generator=gen) for _ in range(P)]
    v.load(sends, m)
    for app in v.ranks:
        app.recv.tensor().fill_(0x5A ^ launch)
        app.recv_counts.fill_(-7)
    torch.cuda.synchronize()
    before = [(app.send.tensor().clone(), app.counts.tensor(torch.int64).clone()) for app in v.ranks]
    tickets = [app.pads.ticket_issued for app in v.ranks]
    v.run_once()
    assert v.verdicts() == [0] * P
    got = v.results()
    want = all_to_all_v_reference(sends, m, R)
    for r, app in enumerate(v.ranks):
        rows, rc = got[r]
        assert rc.tolist() == [m[p][r] for p in range(P)], (launch, r)
        assert torch.equal(rows, want[r].cpu()), (launch, r, rows.shape, want[r].shape)
        tail = app.recv.tensor()[rows.shape[0] * R:]
        assert bool((tail == (0x5A ^ launch)).all()), ("poison past the total", launch, r)
        assert torch.equal(app.send.tensor(), before[r][0]) and torch.equal(app.counts.tensor(torch.int64), before[r][1])
        assert app.pads.ticket_issued == tickets[r] + app.launch_ctas


@pytest.mark.parametrize("row_bytes", ROWS, ids=lambda b: f"{b}B")
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_virtual_ranks_bit_for_bit(algo, world, row_bytes):
    cap = 2 * world * MEAN
    v = VirtualAlltoallv(world, row_bytes, cap, algo)
    try:
        gen = torch.Generator(device="cuda").manual_seed(100 * world + row_bytes)
        hgen = torch.Generator().manual_seed(world + row_bytes)
        launches = 0
        for pattern in PATTERNS:
            for launch in range(3):
                run_and_check(v, counts_for(pattern, world, MEAN, cap, launch, hgen), gen, launch)
                launches += 1
                assert [app.pads.barrier_epoch for app in v.ranks] == [launches] * world
    finally:
        v.close()


@pytest.mark.parametrize("algo", ["push", "pull"])
def test_a_64_mib_exchange(algo):
    P, R = 4, 4096 + 16
    base = (64 << 20) // (P * P * R)
    v = VirtualAlltoallv(P, R, 2 * P * base, algo)
    try:
        gen = torch.Generator(device="cuda").manual_seed(64)
        for launch in range(3):
            m = [[base - (p + q + launch) % 3 for q in range(P)] for p in range(P)]
            run_and_check(v, m, gen, launch)
        assert sum(map(sum, m)) * R > (63 << 20)
    finally:
        v.close()


@pytest.mark.parametrize("world,block_bytes", [(2, 4096), (4, 1 << 20), (8, 48)])
def test_equal_counts_match_the_equal_block_kernel(world, block_bytes):
    R = 16 if block_bytes % 4096 else 4096
    rows = block_bytes // R
    gen = torch.Generator(device="cuda").manual_seed(world)
    sends = [torch.randint(0, 256, (world, block_bytes), dtype=torch.uint8, device="cuda", generator=gen)
             for _ in range(world)]
    eq = VirtualAlltoall(world, block_bytes, "push")
    vv = VirtualAlltoallv(world, R, world * rows, "push")
    try:
        eq.load(sends)
        eq.run_once()
        eq.synchronize()
        vv.load(sends, [[rows] * world for _ in range(world)])
        vv.run_once()
        vv.synchronize()
        for a, b in zip(eq.ranks, vv.ranks):
            assert torch.equal(a.recv.tensor(), b.recv.tensor())
    finally:
        eq.close()
        vv.close()


@pytest.mark.parametrize("rule", [2, 3])
@pytest.mark.parametrize("algo", ["push", "pull"])
def test_refused_counts_move_nothing(algo, rule):
    """Declared capacities are a quarter of what is allocated, so a kernel that ignored the verdict would overwrite
    poison inside its own buffers (and nothing outside them)."""
    P, R, declared = 4, 48, 40
    v = VirtualAlltoallv(P, R, 4 * declared, algo)
    for app in v.ranks:
        app.send_capacity_rows = app.recv_capacity_rows = declared
    try:
        gen = torch.Generator(device="cuda").manual_seed(rule)
        ok = [[declared // P // 2] * P for _ in range(P)]
        bad = [row[:] for row in ok]
        if rule == 2:
            bad[2] = [declared // P + 3] * P          # one rank's row sum above the send capacity
        else:
            for p in range(P):
                bad[p][1] = declared // P + 2         # the column into rank 1 above the receive capacity
        sends = [torch.randint(0, 256, (4 * declared, R), dtype=torch.uint8, device="cuda", generator=gen)
                 for _ in range(P)]
        v.load(sends, bad)
        for app in v.ranks:
            app.recv.tensor().fill_(0xC3)
        torch.cuda.synchronize()
        before = [app.send.tensor().clone() for app in v.ranks]
        v.run_once()
        assert v.verdicts() == [rule] * P
        for r, app in enumerate(v.ranks):
            assert bool((app.recv.tensor() == 0xC3).all()), ("a refused launch wrote data", r)
            assert torch.equal(app.send.tensor(), before[r])
            assert app.recv_counts.tolist() == [bad[p][r] for p in range(P)]
            assert v.ranks[r].C.read_u32(app.pads.status_ptr) == v.ranks[r].C.STATUS_OK
        with pytest.raises(ValueError, match=VERDICT_WORDS[rule]):
            v.results()
        run_and_check(v, ok, gen, 1)
    finally:
        v.close()


def test_exchange_never_synchronises_the_host():
    P, R, n = 4, 64, 200
    v = VirtualAlltoallv(P, R, 2 * n, "push")       # each rank receives about n rows
    try:
        ids = [torch.sort(torch.randint(0, P, (n,), device="cuda")).values for _ in range(P)]
        splits = [torch.bincount(i, minlength=P) for i in ids]
        xs = [torch.randn(n, R // 4, device="cuda") for _ in range(P)]
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            outs = []
            for app, st, x, s in zip(v.ranks, v.streams, xs, splits):
                with torch.cuda.stream(st):
                    outs.append(app.exchange(x, s))
        finally:
            torch.cuda.set_sync_debug_mode(0)
        v.synchronize()
        for app in v.ranks:
            app.check()
        counts = [s.tolist() for s in splits]
        want = all_to_all_v_reference(xs, counts, R)
        for r, (rows, rc) in enumerate(outs):
            assert rc.tolist() == [counts[p][r] for p in range(P)]
            total = sum(rc.tolist())
            assert rows.dtype == torch.float32 and torch.equal(rows[:total].contiguous().view(torch.uint8), want[r])
    finally:
        v.close()


def _cli(bin_dir, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "alltoall"), "-n", "4", "--json", str(rows)] + args, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    got = [json.loads(line) for line in rows.read_text().splitlines()] if rows.exists() else []
    return p, got


@pytest.mark.parametrize("args,variant", [(["--counts", "random"], "push"), (["--counts", "random", "--pull"], "pull"),
                                          (["--counts", "random", "--stock", "memcpy"], "memcpy"),
                                          (["--counts", "skewed", "--row-bytes", "4112"], "push")])
def test_cli_four_ranks(bin_dir, tmp_path, args, variant):
    p, rows = _cli(bin_dir, args + ["--block-bytes", str(1 << 20), "--iters", "3"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    for r in range(4):
        assert f"Passed {r}" in p.stdout, p.stdout
    assert len(rows) == 1 and rows[0]["pattern"] == "alltoallv" and rows[0]["variant"] == variant
    assert rows[0]["mismatches"] == 0 and rows[0]["ms"] > 0 and rows[0]["max_bytes_into_a_rank"] > 0


def test_cli_short_sweep(bin_dir, tmp_path):
    p, rows = _cli(bin_dir, ["--counts", "random", "--sweep", "--block-bytes", str(1 << 18), "--iters", "2"], tmp_path)
    assert p.returncode == 0, p.stdout + p.stderr
    assert [r["block_bytes"] for r in rows] == [16 << k for k in range(15)] and all(r["mismatches"] == 0 for r in rows)
    assert "FAILED" not in p.stdout
