"""Element-wise numerics of the reduce-scatter + all-gather ring (ring_rsag_kernel, csrc/kernels/ring_allreduce.cu) on
virtual ranks of one GPU, modelled on tests/test_gpu_allreduce_numerics.py (whose harness it imports).

Segment s is summed once, by rank s, in a fixed order, and every rank ends with the same bits, so the result must equal
``rsag_expected`` bit for bit for every element type.  VC starts as an all-ones sentinel and must be fully written (the
reduce-scatter phase writes only VC[r] and leaves the rest as it was), receive slots start as a sentinel, VA and 64
guard elements after VC stay untouched, and every status word stays OK.  Each case runs three launches with new data
and advancing epochs; the host synchronises every stream between launches, standing in for the cross-rank barrier.
"""
import os
import subprocess
import sys

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.allreduce_oracle import DTYPES, TORCH_DTYPE, describe, elem_bytes, lanes, make_inputs, mismatches
from tests.rsag_oracle import all_gather_expected, reduce_scatter_expected, rsag_expected, segment
from tests.test_gpu_allreduce_numerics import (CHUNK_VEC, DEV, GUARD, LAUNCHES, _check_untouched, _guard, _max_ctas,
                                              _Ranks)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASE_ID = {"allreduce": 0, "reduce_scatter": 1, "all_gather": 2}


def run_rsag(native, world, dtype, seg_vec, chunk_vec=0, ctas=0, phases="allreduce", data_device="cpu"):
    """Three launches of ring_rsag on ``world`` virtual ranks, ``seg_vec`` 16-byte vectors per segment."""
    td, L, esz = TORCH_DTYPE[dtype], lanes(dtype), elem_bytes(dtype)
    n, chunk_elems = seg_vec * world * L, chunk_vec * L
    n_chunks = native.ring_num_chunks(n // world, chunk_elems, esz)
    ctas = ctas or _max_ctas(world)
    advance = native.rsag_epoch_advance(PHASE_ID[phases], world)
    ranks = _Ranks(world, extra_words=n_chunks)
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric((n + GUARD) * esz, zero=False)
        slots = ranks.symmetric(max(world - 1, 1) * (n // world) * esz, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            vc[r].tensor(td)[n:].copy_(guard)
        epoch = 0
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=400 * world + launch, device=data_device)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor()[:n * esz].fill_(0xFF)        # all-ones: an element nobody writes shows
                slots[r].tensor().fill_(0xFF)               # NaN / all-ones: a slot read before it is written shows
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
                    want = reduce_scatter_expected(vas, r)
                    assert mismatches(vcs[r][seg], want) == 0, \
                        f"launch {launch}, rank {r}: {describe(vcs[r][seg], want, L)}"
                    rest = torch.cat([vcs[r][:seg.start], vcs[r][seg.stop:]])
                    assert bool((rest.view(torch.uint8) == 0xFF).all()), f"rank {r}: VC outside VC[r] was written"
            else:
                want = rsag_expected(vas) if phases == "allreduce" else all_gather_expected(vas)
                for r in range(world):
                    assert mismatches(vcs[r], want) == 0, \
                        f"launch {launch}, rank {r}: {mismatches(vcs[r], want)} wrong, {describe(vcs[r], want, L)}"
                    assert mismatches(vcs[r], vcs[0]) == 0, f"launch {launch}: rank {r} differs from rank 0"
            for r in range(world):
                _check_untouched(va[r], [v.cpu() for v in vas], vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("phases", PHASE_ID)
@pytest.mark.parametrize("world", range(1, 9))
def test_rsag_float_every_world(native, world, phases):
    """1-8 ranks, three full chunks and one vector per segment."""
    run_rsag(native, world, "float", 3 * CHUNK_VEC + 1, phases=phases)


@pytest.mark.parametrize("phases", PHASE_ID)
@pytest.mark.parametrize("dtype", DTYPES)
def test_rsag_every_dtype(native, dtype, phases):
    """Every reference type at 5 ranks, full-range integers (carries, lane widths); the last chunk of a segment is
    513 vectors, fewer than the unrolled body needs."""
    run_rsag(native, 5, dtype, 2 * CHUNK_VEC + 513, phases=phases)


@pytest.mark.parametrize("ctas", ["1", "3", "max"])
@pytest.mark.parametrize("seg_vec,chunk_vec", [(1, 0), (CHUNK_VEC, 0), (1003, 1), (3 * 2049 + 7, 2049)],
                         ids=["one-vector", "one-chunk", "vector-chunks", "body+remainder-chunks"])
def test_rsag_sizes_chunks_and_grids(native, seg_vec, chunk_vec, ctas):
    """Edges of the chunk loop at 5 ranks: one vector per segment; exactly one default chunk per segment; one vector per
    chunk (1003 chunks dealt round-robin); 2049-vector chunks (unrolled body, then a remainder) -- with one CTA, three
    CTAs and the co-residency maximum per rank."""
    run_rsag(native, 5, "float", seg_vec, chunk_vec, 0 if ctas == "max" else int(ctas))


@pytest.mark.parametrize("world", [4, 8])
def test_rsag_large_block(native, world):
    """2^24 + 4P fp32 elements per rank: 2^24/P + 4 per segment, the last chunk of each segment one vector.  Data and
    reference stay on the GPU."""
    run_rsag(native, world, "float", (1 << 22) // world + 1, data_device=f"cuda:{DEV}")


def test_rsag_rejects_overlap_and_bad_sizes(native):
    ranks = _Ranks(2, extra_words=4)
    try:
        buf = ranks.symmetric(4096 * 4)
        p = ranks.pads[0]
        with pytest.raises(Exception, match="overlap"):
            native.ring_rsag(va=buf[0].local_ptr, vc=buf[0].local_ptr + 64, slots_local=0, slots_right=0, vc_right=0,
                             arrived_local=p.chunk_word(0), arrived_right=p.chunk_word(1), rank=0, world=2, n=1024)
        with pytest.raises(Exception, match="16 bytes"):
            native.ring_rsag(va=buf[0].local_ptr, vc=buf[1].local_ptr, slots_local=0, slots_right=0, vc_right=0,
                             arrived_local=p.chunk_word(0), arrived_right=p.chunk_word(1), rank=0, world=2, n=1028)
        with pytest.raises(Exception, match="phases"):
            native.ring_rsag(va=buf[0].local_ptr, vc=buf[1].local_ptr, slots_local=0, slots_right=0, vc_right=0,
                             arrived_local=p.chunk_word(0), arrived_right=p.chunk_word(1), rank=0, world=2, n=1024,
                             phases="broadcast")
    finally:
        ranks.close()


# ---------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("dtype", ["float", "int"])
@pytest.mark.parametrize("world", [4, 5])
def test_virtual_allreduce_ring_rsag(native, world, dtype):
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    n = world * lanes(dtype) * 5003          # a few default chunks per segment, the last one partial
    ar = VirtualAllreduce(world, n, dtype, "ring-rsag")
    try:
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=500 * world + launch)
            ar.load(vas)
            ar.run_once()
            vcs = ar.results()
            want = rsag_expected(vas)
            for r in range(world):
                assert mismatches(vcs[r], want) == 0, f"launch {launch}, rank {r}: {describe(vcs[r], want)}"
            for app, v in zip(ar.ranks, vas):
                assert mismatches(app.va.tensor(v.dtype).cpu(), v) == 0
        assert all(app.launches == LAUNCHES and app.ring_epoch == LAUNCHES * 2 * (world - 1) for app in ar.ranks)
    finally:
        ar.close()


# ------------------------------------------------------------ native CLI ----
def _cli(args, timeout=180, env=None):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    e.update(env or {})
    return subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=timeout, env=e)


@pytest.mark.parametrize("type_", ["float", "int", "double", "short", "uchar"])
@pytest.mark.parametrize("n", [2, 4, 6])
def test_cli_ring_rsag_virtual_ranks(bin_dir, n, type_, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", str(n), "-p", "18", "--iters", "2", "--algo", "ring-rsag",
              "--type", type_, "--json", str(rows)])
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == n and "ring-rsag" in p.stdout
    import json

    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["algo"] == "ring-rsag" and row["ranks"] == n and row["mismatches"] == 0
    assert row["elements"] % (16 // TORCH_DTYPE[type_].itemsize * n) == 0


def test_cli_ring_rsag_profile_relaunch(bin_dir):
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "2", "-p", "18", "--iters", "2", "--algo", "ring-rsag",
              "--profile-relaunch"])
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 2 and "profile relaunch of rank 0 done" in p.stdout


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_torchrun_ring_rsag():
    n = min(torch.cuda.device_count(), 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr",
           "127.0.0.1", "--master-port", "29621", "-m", "hpc_patterns_b200.models.allreduce", "--algo", "ring-rsag",
           "-p", "20", "--iters", "2"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=ROOT))
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert p.stdout.count("Passed") == n and "ring-rsag" in p.stdout
