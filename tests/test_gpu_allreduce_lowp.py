"""bfloat16 / half numerics of the allreduce kernels (csrc/kernels/ring_allreduce.cu) on virtual ranks of one GPU, bit for
bit against tests/lowp_allreduce_oracle.py (harness of tests/test_gpu_allreduce_numerics.py):

* the fused ring (push, push-2slots, pull, pull-2slots) and the accumulate kernel: ``ring_expected``, one add rounded to
  nearest even in the 16-bit type per hop;
* ring-rsag (all three phases): ``rsag_expected`` / ``reduce_scatter_expected`` / ``all_gather_expected``;
* two-shot: ``two_shot_expected``, the fp32 owner-first sum rounded once, the same bits on every rank;
* full-mantissa data, data whose results are subnormal (a flushing adder shows) and, for half, data whose sums reach
  +-inf and NaN (NaN compared by class).

Each case runs three launches with new data; VA and 64 guard elements after VC stay untouched, receive slots and VC start
as an all-ones sentinel, every status word stays OK.  Then the miniapp paths: ``VirtualAllreduce.run_once`` and the
native CLI (``bin/allreduce.bfloat16`` / ``bin/allreduce.half``).
"""
import json
import os
import subprocess
import sys

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.lowp_allreduce_oracle import (LANES, LOWP, TORCH_DTYPE, all_gather_expected, describe, make_inputs,
                                         mismatches, reduce_scatter_expected, ring_expected, rsag_expected, segment,
                                         two_shot_expected)
from tests.test_gpu_allreduce_numerics import CHUNK_VEC, DEV, GUARD, LAUNCHES, RING_VARIANTS, _max_ctas, _Ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ESZ = 2
PHASE_ID = {"allreduce": 0, "reduce_scatter": 1, "all_gather": 2}
KINDS = {"bfloat16": ("full", "subnormal"), "half": ("full", "subnormal", "overflow")}
SIZES = [(1, 0), (CHUNK_VEC, 0), (1003, 1), (3 * 2049 + 7, 2049)]
SIZE_IDS = ["one-vector", "one-chunk", "vector-chunks", "body+remainder-chunks"]


def _guard(dtype):
    return make_inputs(1, GUARD, dtype, seed=0xC0FFEE)[0]


def _check_untouched(va, vas, vc, n, guard, td, rank):
    assert mismatches(va.tensor(td).cpu(), vas[rank].cpu()) == 0, f"rank {rank}: VA changed"
    assert mismatches(vc.tensor(td)[n:].cpu(), guard) == 0, f"rank {rank}: a guard after VC was written"


def _assert_equal(got, want, what):
    k = mismatches(got, want)
    assert k == 0, f"{what}: {k} wrong elements, {describe(got, want)}"


def run_ring(native, world, dtype, variant, nvec, chunk_vec=0, ctas=0, kind="full", data_device="cpu"):
    n_slots, pull = RING_VARIANTS[variant]
    td = TORCH_DTYPE[dtype]
    n, chunk_elems = nvec * LANES, chunk_vec * LANES
    n_chunks = native.ring_num_chunks(n, chunk_elems, ESZ)
    ctas = ctas or _max_ctas(world)
    ranks = _Ranks(world, extra_words=2 * n_chunks)
    try:
        va = ranks.symmetric(n * ESZ)
        vc = ranks.symmetric((n + GUARD) * ESZ, zero=False)
        slots = ranks.symmetric((2 if n_slots == 2 else max(world - 1, 1)) * n * ESZ, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            slots[r].tensor().fill_(0xFF)
            vc[r].tensor(td)[n:].copy_(guard)
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=100 * world + launch, kind=kind, device=data_device)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor(td)[:n].zero_()
            torch.cuda.synchronize(DEV)
            for r in range(world):
                le, ri, p = (r - 1) % world, (r + 1) % world, ranks.pads[r]
                native.ring_allreduce(va[r].local_ptr, vc[r].local_ptr, slots[r].local_ptr, slots[r].ptrs[ri],
                                      p.chunk_word(r), p.chunk_word(ri), world, n, chunk_elems, launch * world,
                                      p.timeout_ns, p.status_ptr, dtype, ctas, DEV, ranks.streams[r].cuda_stream,
                                      n_slots, p.chunk_word(r, n_chunks), p.chunk_word(le, n_chunks), pull,
                                      va[r].ptrs[le], slots[r].ptrs[le])
            ranks.synchronize(native)
            for r in range(world):
                _assert_equal(vc[r].tensor(td)[:n].to(data_device), ring_expected(vas, r), f"launch {launch}, rank {r}")
                _check_untouched(va[r], [v.cpu() for v in vas], vc[r], n, guard, td, r)
    finally:
        ranks.close()


def run_rsag(native, world, dtype, seg_vec, chunk_vec=0, ctas=0, phases="allreduce", kind="full", data_device="cpu"):
    td = TORCH_DTYPE[dtype]
    n, chunk_elems = seg_vec * world * LANES, chunk_vec * LANES
    n_chunks = native.ring_num_chunks(n // world, chunk_elems, ESZ)
    ctas = ctas or _max_ctas(world)
    advance = native.rsag_epoch_advance(PHASE_ID[phases], world)
    ranks = _Ranks(world, extra_words=n_chunks)
    try:
        va = ranks.symmetric(n * ESZ)
        vc = ranks.symmetric((n + GUARD) * ESZ, zero=False)
        slots = ranks.symmetric(max(world - 1, 1) * (n // world) * ESZ, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            vc[r].tensor(td)[n:].copy_(guard)
        epoch = 0
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=400 * world + launch, kind=kind, device=data_device)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor()[:n * ESZ].fill_(0xFF)
                slots[r].tensor().fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                ri, p = (r + 1) % world, ranks.pads[r]
                native.ring_rsag(va=va[r].local_ptr, vc=vc[r].local_ptr, slots_local=slots[r].local_ptr,
                                 slots_right=slots[r].ptrs[ri], vc_right=vc[r].ptrs[ri],
                                 arrived_local=p.chunk_word(r), arrived_right=p.chunk_word(ri), rank=r, world=world,
                                 n=n, chunk_elems=chunk_elems, epoch_base=epoch, timeout_ns=p.timeout_ns,
                                 status=p.status_ptr, dtype=dtype, ctas=ctas, device=DEV,
                                 stream=ranks.streams[r].cuda_stream, phases=phases)
            epoch += advance
            ranks.synchronize(native)
            vcs = [vc[r].tensor(td)[:n].to(data_device) for r in range(world)]
            if phases == "reduce_scatter":
                for r in range(world):
                    seg = segment(n, world, r)
                    _assert_equal(vcs[r][seg], reduce_scatter_expected(vas, r), f"launch {launch}, rank {r}")
                    rest = torch.cat([vcs[r][:seg.start], vcs[r][seg.stop:]])
                    assert bool((rest.view(torch.uint8) == 0xFF).all()), f"rank {r}: VC outside VC[r] was written"
            else:
                want = rsag_expected(vas) if phases == "allreduce" else all_gather_expected(vas)
                for r in range(world):
                    _assert_equal(vcs[r], want, f"launch {launch}, rank {r}")
                    assert bool((vcs[r].view(torch.int16) == vcs[0].view(torch.int16)).all()), f"rank {r} differs"
            for r in range(world):
                _check_untouched(va[r], [v.cpu() for v in vas], vc[r], n, guard, td, r)
    finally:
        ranks.close()


def _block_vec(world):
    return 512 * (4 if world <= 4 else 2)


def run_two_shot(native, world, dtype, slice_vec, ctas=0, kind="full", data_device="cpu"):
    td = TORCH_DTYPE[dtype]
    n = slice_vec * world * LANES
    ctas = ctas or _max_ctas(world)
    ranks = _Ranks(world)
    try:
        va = ranks.symmetric(n * ESZ)
        vc = ranks.symmetric((n + GUARD) * ESZ, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            vc[r].tensor(td)[n:].copy_(guard)
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=200 * world + launch, kind=kind, device=data_device)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor(td)[:n].view(torch.uint8).fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                p = ranks.pads[r]
                p.barrier_epoch += 1
                grid = native.allreduce_two_shot(va[r].ptrs, vc[r].ptrs, p.buf.ptrs, p.ticket_ptr,
                                                 p.ticket_issued & 0xFFFFFFFF, r, n, p.barrier_epoch, p.timeout_ns,
                                                 p.status_ptr, dtype, ctas, DEV, ranks.streams[r].cuda_stream)
                p.advance_tickets(grid)
            ranks.synchronize(native)
            want = two_shot_expected(vas)
            for r in range(world):
                _assert_equal(vc[r].tensor(td)[:n].to(data_device), want, f"launch {launch}, rank {r}")
                _check_untouched(va[r], [v.cpu() for v in vas], vc[r], n, guard, td, r)
    finally:
        ranks.close()


# ------------------------------------------------------------------ the fused ring ----
@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("dtype", LOWP)
def test_ring_every_world(native, dtype, world, variant):
    """1-8 ranks, three full chunks and one vector: acks run in push-2slots from 4 ranks, in pull-2slots from 5."""
    run_ring(native, world, dtype, variant, 3 * CHUNK_VEC + 1)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("dtype,kind", [("bfloat16", "subnormal"), ("half", "subnormal"), ("half", "overflow")])
def test_ring_subnormal_and_overflow(native, dtype, kind, variant):
    """Subnormal results must be kept (a flushing 16-bit adder fails here); fp16 sums that overflow give +-inf and,
    where opposite infinities meet, NaN."""
    run_ring(native, 5, dtype, variant, 2 * CHUNK_VEC + 513, kind=kind)


@pytest.mark.parametrize("ctas", ["1", "3", "max"])
@pytest.mark.parametrize("nvec,chunk_vec", SIZES, ids=SIZE_IDS)
@pytest.mark.parametrize("variant", ["push", "pull-2slots"])
@pytest.mark.parametrize("dtype", LOWP)
def test_ring_sizes_chunks_and_grids(native, dtype, variant, nvec, chunk_vec, ctas):
    run_ring(native, 5, dtype, variant, nvec, chunk_vec, 0 if ctas == "max" else int(ctas))


@pytest.mark.parametrize("dtype", LOWP)
def test_ring_large_block(native, dtype):
    """2^24 + 8 elements per rank at 5 ranks (the last default chunk one vector); reference on the GPU."""
    run_ring(native, 5, dtype, "push", (1 << 21) + 1, data_device=f"cuda:{DEV}")


# -------------------------------------------------------------------- ring-rsag ----
@pytest.mark.parametrize("phases", PHASE_ID)
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("dtype", LOWP)
def test_rsag_every_world(native, dtype, world, phases):
    run_rsag(native, world, dtype, 3 * CHUNK_VEC + 1, phases=phases)


@pytest.mark.parametrize("dtype,kind", [("bfloat16", "subnormal"), ("half", "subnormal"), ("half", "overflow")])
def test_rsag_subnormal_and_overflow(native, dtype, kind):
    run_rsag(native, 5, dtype, 2 * CHUNK_VEC + 513, kind=kind)


@pytest.mark.parametrize("ctas", ["1", "3", "max"])
@pytest.mark.parametrize("seg_vec,chunk_vec", SIZES, ids=SIZE_IDS)
@pytest.mark.parametrize("dtype", LOWP)
def test_rsag_sizes_chunks_and_grids(native, dtype, seg_vec, chunk_vec, ctas):
    run_rsag(native, 5, dtype, seg_vec, chunk_vec, 0 if ctas == "max" else int(ctas))


@pytest.mark.parametrize("dtype", LOWP)
def test_rsag_large_block(native, dtype):
    """2^24 + 8P elements per rank at 4 ranks: 2^22 + 8 per segment."""
    run_rsag(native, 4, dtype, (1 << 21) // 4 + 1, data_device=f"cuda:{DEV}")


# --------------------------------------------------------------------- two-shot ----
SLICES = {"one-vector": lambda w: 1, "below-one-block": lambda w: 37, "one-block": _block_vec,
          "blocks+1": lambda w: 3 * _block_vec(w) + 1}


@pytest.mark.parametrize("slice_", SLICES)
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("dtype", LOWP)
def test_two_shot_every_world(native, dtype, world, slice_):
    """All three <W,U> instantiations one GPU can run (2/4, 4/4, 8/2); tail loop only, main loop only, both."""
    run_two_shot(native, world, dtype, SLICES[slice_](world))


@pytest.mark.parametrize("dtype,kind", [("bfloat16", "subnormal"), ("half", "subnormal"), ("half", "overflow")])
@pytest.mark.parametrize("world", [3, 8])
def test_two_shot_subnormal_and_overflow(native, dtype, kind, world):
    run_two_shot(native, world, dtype, 2 * _block_vec(world) + 5, kind=kind)


@pytest.mark.parametrize("ctas", [1, 3])
@pytest.mark.parametrize("dtype", LOWP)
def test_two_shot_small_grids(native, dtype, ctas):
    run_two_shot(native, 5, dtype, 5 * _block_vec(5) + 3, ctas=ctas)


@pytest.mark.parametrize("dtype", LOWP)
def test_two_shot_large_block(native, dtype):
    """2^24 + 8P elements per rank at 4 ranks."""
    run_two_shot(native, 4, dtype, (1 << 21) // 4 + 1, data_device=f"cuda:{DEV}")


# ------------------------------------------------------------------ accumulate ----
@pytest.mark.parametrize("n", [8, 8 * 1003 + 5, (1 << 20) + 3])
@pytest.mark.parametrize("kind", ["full", "subnormal", "overflow"])
@pytest.mark.parametrize("dtype", LOWP)
def test_accumulate(native, dtype, kind, n):
    """VC += VA: one rounded add per element, the vector body and the scalar tail (n % 8 elements) alike."""
    if kind == "overflow" and dtype == "bfloat16":
        pytest.skip("the overflow data is fp16's")
    td = TORCH_DTYPE[dtype]
    dev = torch.device("cuda", DEV)
    for launch in range(LAUNCHES):
        a, c = make_inputs(2, n, dtype, seed=600 + launch, kind=kind)
        va, vc = a.to(dev), torch.cat([c, _guard(dtype)]).to(dev)
        native.accumulate(va.data_ptr(), vc.data_ptr(), n, dtype, torch.cuda.current_stream(DEV).cuda_stream)
        torch.cuda.synchronize(DEV)
        _assert_equal(vc[:n].cpu(), c + a, f"launch {launch}")
        assert mismatches(vc[n:].cpu(), _guard(dtype)) == 0 and mismatches(va.cpu(), a) == 0


@pytest.mark.parametrize("dtype", LOWP)
def test_init3_and_count_mismatch(native, dtype):
    td = TORCH_DTYPE[dtype]
    n = 8 * 999 + 3
    st = torch.cuda.current_stream(DEV).cuda_stream
    va, vc = (torch.empty(n, dtype=td, device=f"cuda:{DEV}") for _ in range(2))
    native.init3(va.data_ptr(), 0, vc.data_ptr(), n, 3.0, 0.0, 28.0, dtype, st)
    torch.cuda.synchronize(DEV)
    assert bool((va == 3).all()) and bool((vc == 28).all())
    vc[17] = 28.125                           # within 1e-6 of nothing: one mismatch
    count = torch.zeros(1, dtype=torch.int64, device=f"cuda:{DEV}")
    native.count_mismatch(vc.data_ptr(), n, 28.0, dtype, count.data_ptr(), st)
    torch.cuda.synchronize(DEV)
    assert int(count.item()) == 1


# ---------------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("algo", ["ring", "ring-unfused", "ring-rsag", "twoshot"])
@pytest.mark.parametrize("world", [4, 5])
@pytest.mark.parametrize("dtype", LOWP)
def test_virtual_allreduce(native, dtype, world, algo):
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    n = world * LANES * 5003
    ar = VirtualAllreduce(world, n, dtype, algo)
    try:
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=300 * world + launch)
            ar.load(vas)
            ar.run_once()
            vcs = ar.results()
            for r in range(world):
                want = (two_shot_expected(vas) if algo == "twoshot" else rsag_expected(vas) if algo == "ring-rsag"
                        else ring_expected(vas, r))
                _assert_equal(vcs[r], want, f"launch {launch}, rank {r}")
    finally:
        ar.close()


def _cli(args, timeout=180):
    return subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=timeout,
                          env=dict(os.environ, CUDA_VISIBLE_DEVICES="0"))


@pytest.mark.parametrize("args", [["--algo", "ring"], ["--algo", "ring", "--pull"], ["--algo", "ring", "--slots", "2"],
                                  ["--algo", "ring-unfused"], ["--algo", "ring-rsag"], ["-a"]],
                         ids=["ring", "ring-pull", "ring-2slots", "ring-unfused", "ring-rsag", "collective"])
def test_cli_bfloat16(bin_dir, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli([os.path.join(bin_dir, "allreduce.bfloat16"), "-n", "4", "-p", "20", "--iters", "2", "--json", str(rows),
              *args])
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 4 and " bfloat16 " in p.stdout
    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["type"] == "bfloat16" and row["mismatches"] == 0
    assert row["algo"] == ("twoshot" if args == ["-a"] else args[1])


def test_cli_half_ring_rsag_six_ranks(bin_dir):
    p = _cli([os.path.join(bin_dir, "allreduce.half"), "-n", "6", "--algo", "ring-rsag", "-p", "20", "--iters", "2"])
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 6 and "ring-rsag half" in p.stdout


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("args", [["--algo", "ring"], ["--algo", "ring-rsag"], ["-a"]])
@pytest.mark.parametrize("dtype", LOWP)
def test_torchrun_lowp(dtype, args):
    n = min(torch.cuda.device_count(), 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr",
           "127.0.0.1", "--master-port", "29631", "-m", "hpc_patterns_b200.models.allreduce", "--type", dtype, "-p",
           "20", "--iters", "2", *args]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert p.stdout.count("Passed") == n
