"""band / bor / bxor / land / lor / lxor on every allreduce kernel (csrc/kernels/ring_allreduce_ops.cu), bit for bit,
on virtual ranks of one GPU, with the harness of tests/test_gpu_allreduce_numerics.py.

Every result must equal tests/bitop_oracle.py exactly.  VC starts as an all-ones sentinel before every launch (the ops
overwrite VC, so a kernel that reads it shows), receive slots start as a sentinel too, VA and 64 guard elements after
VC stay untouched, and every status word stays OK.  Each case runs three launches, one per input kind: dense random
bits, zero-heavy data, and values nonzero only in their top byte or top 32 bits next to zeros (a logical op that
tests truth per byte or per 32-bit word instead of per element gets those wrong).
"""
import os
import subprocess

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.bitop_oracle import (BIT_OPS, FLOAT_TYPES, INT_TYPES, KINDS, TORCH_DTYPE, allreduce_expected,
                                combine_expected, make_inputs, mismatches, reduce_scatter_expected)
from tests.reduce_op_oracle import describe, elem_bytes, lanes
from tests.rsag_oracle import segment
from tests.test_gpu_allreduce_numerics import CHUNK_VEC, DEV, GUARD, LAUNCHES, RING_VARIANTS, _max_ctas, _Ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(world, n, dtype, seed, launch):
    return make_inputs(world, n, dtype, seed=seed + launch, kind=KINDS[launch % len(KINDS)])


def _guard(dtype):
    return make_inputs(1, GUARD, dtype, seed=0xC0FFEE, kind="dense")[0]


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
            vas = _inputs(world, n, dtype, 100 * world, launch)
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
            want = allreduce_expected(vas, op, dtype)
            for r in range(world):
                got = vc[r].tensor(td)[:n].cpu()
                assert mismatches(got, want) == 0, \
                    f"launch {launch}, rank {r}: {mismatches(got, want)} wrong elements, {describe(got, want, L)}"
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_ring_every_op_and_dtype(native, op, dtype, variant):
    """5 ranks (acks active in both two-slot variants); the last chunk is 513 vectors (remainder loop only)."""
    run_ring(native, 5, dtype, op, variant, 2 * CHUNK_VEC + 513)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op", BIT_OPS)
def test_ring_every_world(native, op, world, variant):
    dtype = INT_TYPES[(world + BIT_OPS.index(op)) % len(INT_TYPES)]
    run_ring(native, world, dtype, op, variant, 3 * CHUNK_VEC + 1)


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
            vas = _inputs(world, n, dtype, 400 * world, launch)
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
                want = allreduce_expected(vas, op, dtype)
                for r in range(world):
                    assert mismatches(vcs[r], want) == 0, \
                        f"launch {launch}, rank {r}: {mismatches(vcs[r], want)} wrong, {describe(vcs[r], want, L)}"
            for r in range(world):
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("phases", PHASE_ID)
@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_rsag_every_op_and_dtype(native, op, dtype, phases):
    run_rsag(native, 5, dtype, op, 2 * CHUNK_VEC + 513, phases=phases)


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op", BIT_OPS)
def test_rsag_every_world(native, op, world):
    dtype = INT_TYPES[(world + BIT_OPS.index(op)) % len(INT_TYPES)]
    run_rsag(native, world, dtype, op, 3 * CHUNK_VEC + 1)


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
            vas = _inputs(world, n, dtype, 200 * world, launch)
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
            want = allreduce_expected(vas, op, dtype)
            for r in range(world):
                got = vc[r].tensor(td)[:n].cpu()
                assert mismatches(got, want) == 0, \
                    f"launch {launch}, rank {r}: {mismatches(got, want)} wrong, {describe(got, want, L)}"
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_two_shot_every_op_and_dtype(native, op, dtype):
    """4 ranks, k blocks + 1 vector per slice: the main blocks and the tail loop."""
    run_two_shot(native, 4, dtype, op, 2 * _block_vec(4) + 1)


@pytest.mark.parametrize("slice_", ["below-one-block", "blocks+tail"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("op", BIT_OPS)
def test_two_shot_every_width(native, op, world, slice_):
    """The <W,U> = 2/4, 4/4, 8/2 instantiations; the tail loop alone, and blocks + tail."""
    dtype = INT_TYPES[(world + BIT_OPS.index(op)) % len(INT_TYPES)]
    run_two_shot(native, world, dtype, op, 37 if slice_ == "below-one-block" else 3 * _block_vec(world) + 1)


# ------------------------------------------------------------------ combine ----
@pytest.mark.parametrize("dtype", INT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_combine(native, op, dtype):
    """VC = op(VC, VA) over whole vectors and a partial last vector; nothing after the n elements is written."""
    L = lanes(dtype)
    for i, n in enumerate((L * 3000 + L - 1, L - 1 if L > 1 else 1, L * 777)):
        vc0, va = make_inputs(2, n + GUARD, dtype, seed=600 + i, kind=KINDS[i])
        vc = vc0.clone().to(f"cuda:{DEV}")
        va_d = va.to(f"cuda:{DEV}")
        native.accumulate(va_d.data_ptr(), vc.data_ptr(), n, dtype, torch.cuda.current_stream(DEV).cuda_stream, op=op)
        torch.cuda.synchronize(DEV)
        got = vc.cpu()
        want = combine_expected(vc0[:n], va[:n], op, dtype)
        assert mismatches(got[:n], want) == 0, f"n={n}: {describe(got[:n], want, L)}"
        assert mismatches(got[n:], vc0[n:]) == 0, f"n={n}: elements after n were written"
        assert mismatches(va_d.cpu(), va) == 0


# ------------------------------------------------------- the float refusal ----
@pytest.mark.parametrize("dtype", FLOAT_TYPES)
@pytest.mark.parametrize("op", BIT_OPS)
def test_every_binding_refuses_floating_types(native, op, dtype):
    """Refused before any kernel is chosen, with one message that names the op and the type."""
    world, esz = 2, elem_bytes(dtype)
    n = 64 * world
    msg = f"op must be sum, prod, min or max for .*{op} reduces integer types only"
    ranks = _Ranks(world, extra_words=4)
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric(n * esz)
        slots = ranks.symmetric(n * esz)
        p = ranks.pads[0]
        st = ranks.streams[0].cuda_stream
        with pytest.raises(Exception, match=msg):
            native.ring_allreduce(va[0].local_ptr, vc[0].local_ptr, slots[0].local_ptr, slots[0].ptrs[1],
                                  p.chunk_word(0), p.chunk_word(1), world, n, 0, 0, p.timeout_ns, p.status_ptr, dtype,
                                  1, DEV, st, op=op)
        with pytest.raises(Exception, match=msg):
            native.ring_rsag(va=va[0].local_ptr, vc=vc[0].local_ptr, slots_local=slots[0].local_ptr,
                             slots_right=slots[0].ptrs[1], vc_right=vc[0].ptrs[1], arrived_local=p.chunk_word(0),
                             arrived_right=p.chunk_word(1), rank=0, world=world, n=n, timeout_ns=p.timeout_ns,
                             status=p.status_ptr, dtype=dtype, ctas=1, device=DEV, stream=st, op=op)
        with pytest.raises(Exception, match=msg):
            native.allreduce_two_shot(va[0].ptrs, vc[0].ptrs, p.buf.ptrs, p.ticket_ptr, 0, 0, n, 1, p.timeout_ns,
                                      p.status_ptr, dtype, 1, DEV, st, op=op)
        with pytest.raises(Exception, match=msg):
            native.accumulate(va[0].local_ptr, vc[0].local_ptr, n, dtype, st, op=op)
        torch.cuda.synchronize(DEV)
        assert [native.read_u32(q.status_ptr) for q in ranks.pads] == [native.STATUS_OK] * world
    finally:
        ranks.close()


# --------------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("dtype", ["int", "ulong", "ushort", "uchar"])
@pytest.mark.parametrize("algo,slots,pull", [("ring", 0, False), ("ring", 2, True), ("twoshot", 0, False),
                                             ("ring-unfused", 0, False), ("ring-rsag", 0, False)],
                         ids=["ring", "ring-pull-2slots", "twoshot", "ring-unfused", "ring-rsag"])
@pytest.mark.parametrize("op", BIT_OPS)
def test_virtual_allreduce_bitops(native, op, algo, slots, pull, dtype):
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    world = 5
    n = world * lanes(dtype) * 5003
    ar = VirtualAllreduce(world, n, dtype, algo, slots=slots, pull=pull, op=op)
    try:
        for launch in range(LAUNCHES):
            vas = _inputs(world, n, dtype, 300 * world, launch)
            ar.load(vas)
            for app in ar.ranks:
                app.vc.tensor().fill_(0xFF)
            torch.cuda.synchronize(DEV)
            ar.run_once()
            vcs = ar.results()
            want = allreduce_expected(vas, op, dtype)
            for r in range(world):
                assert mismatches(vcs[r], want) == 0, f"launch {launch}, rank {r}: {describe(vcs[r], want)}"
    finally:
        ar.close()


@pytest.mark.parametrize("op", BIT_OPS)
def test_virtual_allreduce_constant_check(native, op):
    """run()'s initialisation: the op's own constant-data check passes on every rank."""
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    ar = VirtualAllreduce(4, 4 * 16 * 1000, "uchar", "ring", op=op)
    try:
        for app in ar.ranks:
            app.initialize()
        torch.cuda.synchronize(DEV)
        ar.run_once()
        ar.synchronize()
        assert all(app.mismatches() == 0 for app in ar.ranks)
    finally:
        ar.close()


# ------------------------------------------------------------- native CLI ----
def _cli(args, timeout=180):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    return subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=timeout, env=e)


@pytest.mark.parametrize("name,args", [
    ("allreduce.int", ["--op", "land"]),
    ("allreduce", ["--type", "uchar", "-a", "--op", "bxor"]),
    ("allreduce.long", ["--algo", "ring-rsag", "--op", "bor"]),
    ("allreduce", ["--type", "ushort", "--slots", "2", "--pull", "--op", "lxor"]),
    ("allreduce", ["--type", "short", "--algo", "ring-unfused", "--op", "band"]),
    ("allreduce", ["--type", "ulong", "-R", "--op", "lor"]),
    ("allreduce", ["--type", "uint", "-H", "--op", "bxor"]),
    ("allreduce", ["--type", "uchar", "-S", "-a", "--op", "land"]),
], ids=["int-land", "uchar-a-bxor", "long-rsag-bor", "ushort-pull-2slots-lxor", "short-unfused-band", "ulong-R-lor",
        "uint-H-bxor", "uchar-S-a-land"])
def test_cli_bitops(bin_dir, name, args, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = _cli([os.path.join(bin_dir, name), "-n", "4", "-p", "18", "--iters", "2", "--json", str(rows)] + args)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 4, p.stdout
    import json

    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["op"] == args[-1] and row["mismatches"] == 0
    if "-a" in args:
        assert row["algo"] == "twoshot" and "NVLS reduces sums only" in p.stdout


def test_cli_refusals(bin_dir):
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "2", "-p", "12", "-a", "--coll", "nvls", "--type", "int",
              "--op", "band"])
    assert p.returncode != 0 and "sum-only" in p.stderr
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "2", "-p", "12", "--op", "band"])    # float by default
    assert p.returncode != 0 and "integer types only" in p.stderr and "Passed" not in p.stdout
