"""prod / min / max on every allreduce kernel (csrc/kernels/ring_allreduce_ops.cu), bit for bit, on virtual ranks of
one GPU, with the harness of tests/test_gpu_allreduce_numerics.py.

Every result must equal tests/reduce_op_oracle.py exactly, NaN included (results are canonical NaNs).  VC starts as an
all-ones sentinel before every launch: the op kernels overwrite VC, so a kernel that reads VC before writing it shows.
Receive slots start as a sentinel too, VA and 64 guard elements after VC stay untouched, and every status word stays
OK.  Each case runs three launches with new data of the input kinds that apply to (op, type), one kind per launch:
signed and unsigned extremes, +-0 / +-inf / NaN, duplicates, products near 1, subnormal products and overflowing ones.
"""
import os
import subprocess

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.reduce_op_oracle import (OPS, TORCH_DTYPE, TYPES, combine_expected, describe, elem_bytes, kinds, lanes,
                                    make_inputs, mismatches, reduce_scatter_expected, ring_expected, rsag_expected,
                                    two_shot_expected)
from tests.rsag_oracle import segment
from tests.test_gpu_allreduce_numerics import CHUNK_VEC, DEV, GUARD, LAUNCHES, RING_VARIANTS, _max_ctas, _Ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(world, n, dtype, op, seed, launch):
    k = kinds(op, dtype)
    return make_inputs(world, n, dtype, seed=seed + launch, op=op, kind=k[launch % len(k)])


def _guard(dtype):
    return make_inputs(1, GUARD, dtype, seed=0xC0FFEE, op="max", kind=kinds("max", dtype)[0])[0]


def _check_untouched(va, vas, vc, n, guard, td, rank):
    assert mismatches(va.tensor(td).cpu(), vas[rank]) == 0, f"rank {rank}: VA changed"
    assert mismatches(vc.tensor(td)[n:].cpu(), guard) == 0, f"rank {rank}: a guard after VC was written"


def run_ring(native, world, dtype, op, variant, nvec, chunk_vec=0, ctas=0):
    n_slots, pull = RING_VARIANTS[variant]
    td, L, esz = TORCH_DTYPE[dtype], lanes(dtype), elem_bytes(dtype)
    n, chunk_elems = nvec * L, chunk_vec * L
    n_chunks = native.ring_num_chunks(n, chunk_elems, esz)
    ctas = ctas or _max_ctas(world)
    ranks = _Ranks(world, extra_words=2 * n_chunks)
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric((n + GUARD) * esz, zero=False)
        slots = ranks.symmetric((2 if n_slots == 2 else max(world - 1, 1)) * n * esz, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            slots[r].tensor().fill_(0xFF)
            vc[r].tensor(td)[n:].copy_(guard)
        for launch in range(LAUNCHES):
            vas = _inputs(world, n, dtype, op, 100 * world, launch)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor()[:n * esz].fill_(0xFF)        # the op kernels must overwrite VC, never read it
            torch.cuda.synchronize(DEV)
            for r in range(world):
                le, ri, p = (r - 1) % world, (r + 1) % world, ranks.pads[r]
                native.ring_allreduce(va[r].local_ptr, vc[r].local_ptr, slots[r].local_ptr, slots[r].ptrs[ri],
                                      p.chunk_word(r), p.chunk_word(ri), world, n, chunk_elems, launch * world,
                                      p.timeout_ns, p.status_ptr, dtype, ctas, DEV, ranks.streams[r].cuda_stream,
                                      n_slots, p.chunk_word(r, n_chunks), p.chunk_word(le, n_chunks), pull,
                                      va[r].ptrs[le], slots[r].ptrs[le], op=op)
            ranks.synchronize(native)
            for r in range(world):
                got, want = vc[r].tensor(td)[:n].cpu(), ring_expected(vas, r, op, dtype)
                assert mismatches(got, want) == 0, \
                    f"launch {launch}, rank {r}: {mismatches(got, want)} wrong elements, {describe(got, want, L)}"
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("op", OPS)
def test_ring_every_op_and_dtype(native, op, dtype, variant):
    """5 ranks (acks active in both two-slot variants); the last chunk is 513 vectors (remainder loop only)."""
    run_ring(native, 5, dtype, op, variant, 2 * CHUNK_VEC + 513)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op", OPS)
def test_ring_every_world(native, op, world, variant):
    run_ring(native, world, "float", op, variant, 3 * CHUNK_VEC + 1)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("nvec,chunk_vec,ctas", [(1, 0, 0), (1003, 1, 3), (3 * 2049 + 7, 2049, 1)],
                         ids=["one-vector", "vector-chunks", "body+remainder-chunks"])
def test_ring_sizes_chunks_and_grids(native, nvec, chunk_vec, ctas, variant):
    run_ring(native, 5, "half", "max", variant, nvec, chunk_vec, ctas)


# ---------------------------------------------------------------- ring-rsag ----
PHASE_ID = {"allreduce": 0, "reduce_scatter": 1}


def run_rsag(native, world, dtype, op, seg_vec, chunk_vec=0, ctas=0, phases="allreduce"):
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
            vas = _inputs(world, n, dtype, op, 400 * world, launch)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor()[:n * esz].fill_(0xFF)
                slots[r].tensor().fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                ri, p = (r + 1) % world, ranks.pads[r]
                native.ring_rsag(va=va[r].local_ptr, vc=vc[r].local_ptr, slots_local=slots[r].local_ptr,
                                 slots_right=slots[r].ptrs[ri], vc_right=vc[r].ptrs[ri],
                                 arrived_local=p.chunk_word(r), arrived_right=p.chunk_word(ri), rank=r, world=world,
                                 n=n, chunk_elems=chunk_elems, epoch_base=epoch, timeout_ns=p.timeout_ns,
                                 status=p.status_ptr, dtype=dtype, ctas=ctas, device=DEV,
                                 stream=ranks.streams[r].cuda_stream, phases=phases, op=op)
            epoch += advance
            ranks.synchronize(native)
            vcs = [vc[r].tensor(td)[:n].cpu() for r in range(world)]
            if phases == "reduce_scatter":
                for r in range(world):
                    seg = segment(n, world, r)
                    want = reduce_scatter_expected(vas, r, op, dtype)
                    assert mismatches(vcs[r][seg], want) == 0, \
                        f"launch {launch}, rank {r}: {describe(vcs[r][seg], want, L)}"
                    rest = torch.cat([vcs[r][:seg.start], vcs[r][seg.stop:]])
                    assert bool((rest.view(torch.uint8) == 0xFF).all()), f"rank {r}: VC outside VC[r] was written"
            else:
                want = rsag_expected(vas, op, dtype)
                for r in range(world):
                    assert mismatches(vcs[r], want) == 0, \
                        f"launch {launch}, rank {r}: {mismatches(vcs[r], want)} wrong, {describe(vcs[r], want, L)}"
            for r in range(world):
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("phases", PHASE_ID)
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("op", OPS)
def test_rsag_every_op_and_dtype(native, op, dtype, phases):
    run_rsag(native, 5, dtype, op, 2 * CHUNK_VEC + 513, phases=phases)


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op", OPS)
def test_rsag_every_world(native, op, world):
    run_rsag(native, world, "float", op, 3 * CHUNK_VEC + 1)


@pytest.mark.parametrize("seg_vec,chunk_vec,ctas", [(1, 0, 0), (1003, 1, 3), (3 * 2049 + 7, 2049, 1)],
                         ids=["one-vector", "vector-chunks", "body+remainder-chunks"])
def test_rsag_sizes_chunks_and_grids(native, seg_vec, chunk_vec, ctas):
    run_rsag(native, 5, "bfloat16", "prod", seg_vec, chunk_vec, ctas)


# ----------------------------------------------------------------- two-shot ----
def _block_vec(world):
    return 512 * (4 if world <= 4 else 2)


def run_two_shot(native, world, dtype, op, slice_vec, ctas=0):
    td, L, esz = TORCH_DTYPE[dtype], lanes(dtype), elem_bytes(dtype)
    n = slice_vec * world * L
    ctas = ctas or _max_ctas(world)
    ranks = _Ranks(world)
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric((n + GUARD) * esz, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            vc[r].tensor(td)[n:].copy_(guard)
        for launch in range(LAUNCHES):
            vas = _inputs(world, n, dtype, op, 200 * world, launch)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor()[:n * esz].fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                p = ranks.pads[r]
                p.barrier_epoch += 1
                grid = native.allreduce_two_shot(va[r].ptrs, vc[r].ptrs, p.buf.ptrs, p.ticket_ptr,
                                                 p.ticket_issued & 0xFFFFFFFF, r, n, p.barrier_epoch, p.timeout_ns,
                                                 p.status_ptr, dtype, ctas, DEV, ranks.streams[r].cuda_stream, op=op)
                p.advance_tickets(grid)
            ranks.synchronize(native)
            want = two_shot_expected(vas, op, dtype)
            for r in range(world):
                got = vc[r].tensor(td)[:n].cpu()
                assert mismatches(got, want) == 0, \
                    f"launch {launch}, rank {r}: {mismatches(got, want)} wrong, {describe(got, want, L)}"
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("world", [2, 4, 5])
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("op", OPS)
def test_two_shot_every_op_and_dtype(native, op, dtype, world):
    """Every <W,U> instantiation up to 8 ranks (2/4, 4/4, 8/2); k blocks + 1 vector per slice: the main blocks and the
    tail loop, both owner first."""
    run_two_shot(native, world, dtype, op, 2 * _block_vec(world) + 1)


@pytest.mark.parametrize("slice_", ["below-one-block", "blocks+1"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("op", OPS)
def test_two_shot_every_width(native, op, world, slice_):
    """The <W,U> = 2/4, 4/4, 8/2 instantiations; the tail loop alone, and blocks + tail."""
    dtype = "bfloat16" if op == "prod" else "float"      # 16-bit prod: the fp32 kernel
    run_two_shot(native, world, dtype, op, 37 if slice_ == "below-one-block" else 3 * _block_vec(world) + 1)


@pytest.mark.parametrize("world", [2, 5])
def test_two_shot_small_grid(native, world):
    run_two_shot(native, world, "double", "min", 5 * _block_vec(world) + 3, ctas=1)


# ------------------------------------------------------------------ combine ----
@pytest.mark.parametrize("dtype", TYPES)
@pytest.mark.parametrize("op", OPS)
def test_combine(native, op, dtype):
    """VC = op(VC, VA) over whole vectors and a partial last vector; nothing after the n elements is written."""
    td, L, esz = TORCH_DTYPE[dtype], lanes(dtype), elem_bytes(dtype)
    for n in (L * 3000 + L - 1, L - 1 if L > 1 else 1, L * 777):
        vc0, va = _inputs(2, n + GUARD, dtype, op, 600, n % 3)
        vc = vc0.clone().to(f"cuda:{DEV}")
        va_d = va.to(f"cuda:{DEV}")
        native.accumulate(va_d.data_ptr(), vc.data_ptr(), n, dtype, torch.cuda.current_stream(DEV).cuda_stream, op=op)
        torch.cuda.synchronize(DEV)
        got = vc.cpu()
        want = combine_expected(vc0[:n], va[:n], op, dtype)
        assert mismatches(got[:n], want) == 0, f"n={n}: {describe(got[:n], want, L)}"
        assert mismatches(got[n:], vc0[n:]) == 0, f"n={n}: elements after n were written"
        assert mismatches(va_d.cpu(), va) == 0


def test_accumulate_rejects_unknown_op(native):
    with pytest.raises(Exception, match="op must be"):
        native.accumulate(0, 0, 0, "float", 0, op="avg")


# --------------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("dtype", ["float", "ushort", "bfloat16", "long"])
@pytest.mark.parametrize("algo,slots,pull", [("ring", 0, False), ("ring", 2, True), ("twoshot", 0, False),
                                             ("ring-unfused", 0, False), ("ring-rsag", 0, False)],
                         ids=["ring", "ring-pull-2slots", "twoshot", "ring-unfused", "ring-rsag"])
@pytest.mark.parametrize("op", OPS)
def test_virtual_allreduce_ops(native, op, algo, slots, pull, dtype):
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    world = 5
    n = world * lanes(dtype) * 5003
    ar = VirtualAllreduce(world, n, dtype, algo, slots=slots, pull=pull, op=op)
    try:
        for launch in range(LAUNCHES):
            vas = _inputs(world, n, dtype, op, 300 * world, launch)
            ar.load(vas)
            for app in ar.ranks:
                app.vc.tensor().fill_(0xFF)
            torch.cuda.synchronize(DEV)
            ar.run_once()
            vcs = ar.results()
            for r in range(world):
                want = (two_shot_expected(vas, op, dtype) if algo == "twoshot"
                        else rsag_expected(vas, op, dtype) if algo == "ring-rsag"
                        else ring_expected(vas, r, op, dtype))
                assert mismatches(vcs[r], want) == 0, f"launch {launch}, rank {r}: {describe(vcs[r], want)}"
    finally:
        ar.close()


@pytest.mark.parametrize("op", OPS)
def test_virtual_allreduce_constant_check(native, op):
    """run(): the op's own constant-data check passes on every rank."""
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce, expected_value, op_input

    ar = VirtualAllreduce(4, 4 * 8 * 1000, "half", "ring", op=op)
    try:
        for app in ar.ranks:
            app.initialize()
        torch.cuda.synchronize(DEV)
        ar.run_once()
        ar.synchronize()
        assert all(app.mismatches() == 0 for app in ar.ranks)
        assert expected_value(4, op) == {"max": 3, "min": 1, "prod": 4}[op]
        assert [op_input(op, r, 4) for r in range(4)] == {"max": [0, 1, 2, 3], "min": [4, 3, 2, 1],
                                                          "prod": [1, 2, 1, 2]}[op]
    finally:
        ar.close()


def test_nvls_refuses_ops(native):
    with pytest.raises(Exception, match="sum"):
        native.allreduce_nvls(0, 0, [0, 0], 0, 0, 0, 64, 1, op="max")


# ------------------------------------------------------------- native CLI ----
def _cli(args, timeout=180):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    return subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=timeout, env=e)


@pytest.mark.parametrize("op", ["max", "min", "prod"])
@pytest.mark.parametrize("args", [["--type", "float"], ["--type", "ushort", "--algo", "ring-rsag"],
                                  ["--type", "bfloat16", "-a"], ["--type", "long", "--slots", "2", "--pull"],
                                  ["--type", "uchar", "--algo", "ring-unfused"], ["--type", "short", "-R"],
                                  ["--type", "half", "-a", "-S"], ["--type", "int", "-H"]],
                         ids=["float", "ushort-rsag", "bf16-a", "long-pull-2slots", "uchar-unfused", "short-R",
                              "half-a-S", "int-H"])
def test_cli_ops(bin_dir, op, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "4", "-p", "18", "--iters", "2", "--op", op,
              "--json", str(rows)] + args)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 4, p.stdout
    import json

    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["op"] == op and row["mismatches"] == 0
    if "-a" in args:
        assert row["algo"] == "twoshot" and "NVLS reduces sums only" in p.stdout


def test_cli_nvls_op_refused(bin_dir):
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "2", "-p", "12", "-a", "--coll", "nvls", "--op", "max"])
    assert p.returncode != 0 and "sum-only" in p.stderr
