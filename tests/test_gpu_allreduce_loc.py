"""maxloc / minloc on every allreduce kernel (csrc/kernels/ring_allreduce_ops.cu) for the five value-index pair types,
bit for bit against tests/loc_oracle.py, on virtual ranks of one GPU.

Inputs: values from a tiny set (heavy ties), signed zeros, ±inf and NaNs of both signs and several payloads, and
indices that include INT_MIN, INT_MAX and negatives; the padding bytes of VA hold garbage.  VC and the receive slots
start as an all-ones sentinel (the ops overwrite VC, so a kernel that reads it shows), VA and GUARD pairs after VC stay
untouched, and every status word stays OK.
"""
import os
import random
import subprocess

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.loc_oracle import (KINDS, LOC_OPS, PAIR_TYPES, allreduce_expected, combine_expected, describe, make_inputs,
                              mismatches, pair_bytes, pairs_per_vector)
from tests.test_gpu_allreduce_numerics import DEV, GUARD, RING_VARIANTS, _max_ctas, _Ranks

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _u8(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8)


def _bytes(t):
    return t.cpu().numpy().tobytes()


def _guard(dtype):
    """GUARD pairs' worth of random bytes placed after every VC: no kernel may write them."""
    rng = random.Random(0xC0FFEE)
    return bytes(rng.randrange(256) for _ in range(GUARD * pair_bytes(dtype)))


def _vc_with_guard(ranks, n, dtype):
    esz = pair_bytes(dtype)
    vc = ranks.symmetric((n + GUARD) * esz, zero=False)
    guard = _guard(dtype)
    for b in vc:
        b.tensor(torch.uint8)[n * esz:].copy_(_u8(guard))
    return vc, guard


def _check(vc, va, vas, want, n, dtype, guard, what):
    """VC = want on every rank, VA untouched, the guard after VC untouched."""
    esz = pair_bytes(dtype)
    for r in range(len(vas)):
        got = _bytes(vc[r].tensor(torch.uint8))
        assert mismatches(got[:n * esz], want, dtype) == 0, f"{what}, rank {r}: {describe(got[:n * esz], want, dtype)}"
        assert got[n * esz:] == guard, f"{what}, rank {r}: a guard after VC was written"
        assert _bytes(va[r].tensor(torch.uint8)) == vas[r], f"{what}, rank {r}: VA changed"


def run_ring(native, world, dtype, op, variant, nvec, chunk_vec=0):
    """The fused ring (push / pull, P-1 or two slots); VC and the slots start as an all-ones sentinel."""
    n_slots, pull = RING_VARIANTS[variant]
    L, esz = pairs_per_vector(dtype), pair_bytes(dtype)
    n, chunk_elems = nvec * L, chunk_vec * L
    n_chunks = native.ring_num_chunks(n, chunk_elems, esz)
    ranks = _Ranks(world, extra_words=2 * n_chunks)
    try:
        va = ranks.symmetric(n * esz)
        vc, guard = _vc_with_guard(ranks, n, dtype)
        slots = ranks.symmetric((2 if n_slots == 2 else max(world - 1, 1)) * n * esz, zero=False)
        for launch, kind in enumerate(KINDS):
            vas = make_inputs(world, n, dtype, seed=100 * world + launch, kind=kind)
            for r in range(world):
                va[r].tensor(torch.uint8).copy_(_u8(vas[r]))          # garbage padding bytes included
                vc[r].tensor(torch.uint8)[:n * esz].fill_(0xFF)        # overwritten, never read
                slots[r].tensor(torch.uint8).fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                le, ri, p = (r - 1) % world, (r + 1) % world, ranks.pads[r]
                native.ring_allreduce(va[r].local_ptr, vc[r].local_ptr, slots[r].local_ptr, slots[r].ptrs[ri],
                                      p.chunk_word(r), p.chunk_word(ri), world, n, chunk_elems, launch * world,
                                      p.timeout_ns, p.status_ptr, dtype, _max_ctas(world), DEV,
                                      ranks.streams[r].cuda_stream, n_slots, p.chunk_word(r, n_chunks),
                                      p.chunk_word(le, n_chunks), pull, va[r].ptrs[le], slots[r].ptrs[le], op=op)
            ranks.synchronize(native)                                  # status words OK
            _check(vc, va, vas, allreduce_expected(op, vas, dtype), n, dtype, guard, f"{variant} {kind}")
    finally:
        ranks.close()


def run_rsag(native, world, dtype, op, seg_vec, chunk_vec=0):
    L, esz = pairs_per_vector(dtype), pair_bytes(dtype)
    n, chunk_elems = seg_vec * world * L, chunk_vec * L
    n_chunks = native.ring_num_chunks(n // world, chunk_elems, esz)
    advance = native.rsag_epoch_advance(native.RSAG_ALLREDUCE, world)
    ranks = _Ranks(world, extra_words=n_chunks)
    try:
        va = ranks.symmetric(n * esz)
        vc, guard = _vc_with_guard(ranks, n, dtype)
        slots = ranks.symmetric(max(world - 1, 1) * (n // world) * esz, zero=False)
        for launch, kind in enumerate(KINDS):
            vas = make_inputs(world, n, dtype, seed=400 * world + launch, kind=kind)
            for r in range(world):
                va[r].tensor(torch.uint8).copy_(_u8(vas[r]))
                vc[r].tensor(torch.uint8)[:n * esz].fill_(0xFF)
                slots[r].tensor(torch.uint8).fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                ri, p = (r + 1) % world, ranks.pads[r]
                native.ring_rsag(va=va[r].local_ptr, vc=vc[r].local_ptr, slots_local=slots[r].local_ptr,
                                 slots_right=slots[r].ptrs[ri], vc_right=vc[r].ptrs[ri],
                                 arrived_local=p.chunk_word(r), arrived_right=p.chunk_word(ri), rank=r, world=world,
                                 n=n, chunk_elems=chunk_elems, epoch_base=launch * advance, timeout_ns=p.timeout_ns,
                                 status=p.status_ptr, dtype=dtype, ctas=_max_ctas(world), device=DEV,
                                 stream=ranks.streams[r].cuda_stream, op=op)
            ranks.synchronize(native)
            _check(vc, va, vas, allreduce_expected(op, vas, dtype), n, dtype, guard, f"rsag {kind}")
    finally:
        ranks.close()


def _block_vec(world):
    return 512 * (4 if world <= 4 else 2)


def run_two_shot(native, world, dtype, op, slice_vec):
    L, esz = pairs_per_vector(dtype), pair_bytes(dtype)
    n = slice_vec * world * L
    ranks = _Ranks(world)
    try:
        va = ranks.symmetric(n * esz)
        vc, guard = _vc_with_guard(ranks, n, dtype)
        for launch, kind in enumerate(KINDS):
            vas = make_inputs(world, n, dtype, seed=200 * world + launch, kind=kind)
            for r in range(world):
                va[r].tensor(torch.uint8).copy_(_u8(vas[r]))
                vc[r].tensor(torch.uint8)[:n * esz].fill_(0xFF)
            torch.cuda.synchronize(DEV)
            for r in range(world):
                p = ranks.pads[r]
                p.barrier_epoch += 1
                grid = native.allreduce_two_shot(va[r].ptrs, vc[r].ptrs, p.buf.ptrs, p.ticket_ptr,
                                                 p.ticket_issued & 0xFFFFFFFF, r, n, p.barrier_epoch, p.timeout_ns,
                                                 p.status_ptr, dtype, _max_ctas(world), DEV,
                                                 ranks.streams[r].cuda_stream, op=op)
                p.advance_tickets(grid)
            ranks.synchronize(native)
            _check(vc, va, vas, allreduce_expected(op, vas, dtype), n, dtype, guard, f"two-shot {kind}")
    finally:
        ranks.close()


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_ring_every_type(native, op, dtype, variant):
    """5 ranks (acks active in both two-slot variants); small chunks, the last one partial."""
    run_ring(native, 5, dtype, op, variant, 5 * 64 + 37, chunk_vec=64)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("world", [1, 2, 3, 4, 6, 8])
@pytest.mark.parametrize("op", LOC_OPS)
def test_ring_every_world(native, op, world, variant):
    dtype = PAIR_TYPES[(world + LOC_OPS.index(op)) % len(PAIR_TYPES)]
    run_ring(native, world, dtype, op, variant, 2 * 256 + 37, chunk_vec=256)


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_rsag_every_type(native, op, dtype):
    run_rsag(native, 5, dtype, op, 3 * 64 + 17, chunk_vec=64)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 6, 8])
@pytest.mark.parametrize("op", LOC_OPS)
def test_rsag_every_world(native, op, world):
    dtype = PAIR_TYPES[(world + LOC_OPS.index(op)) % len(PAIR_TYPES)]
    run_rsag(native, world, dtype, op, 3 * 64 + 5, chunk_vec=64)


@pytest.mark.parametrize("slice_", ["below-one-block", "blocks+tail"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_two_shot_every_shape(native, op, dtype, world, slice_):
    """Every op x pair type on the <W,U> = 2/4, 4/4 and 8/2 instantiations: the tail loop alone, and blocks + tail."""
    run_two_shot(native, world, dtype, op, 37 if slice_ == "below-one-block" else _block_vec(world) + 1)


# ------------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("variant", [("ring", 0, False), ("ring", 2, True), ("ring-unfused", 0, False),
                                     ("ring-rsag", 0, False), ("twoshot", 0, False)],
                         ids=["ring", "ring-pull-2slots", "ring-unfused", "ring-rsag", "twoshot"])
@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_virtual_allreduce(op, dtype, variant):
    """``VirtualAllreduce``: load() takes and results() gives (values, indices) per rank; VC from an all-ones sentinel."""
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce
    from hpc_patterns_b200.ops.allreduce import pack_loc, unpack_loc

    algo, slots, pull = variant
    world = 5
    n = world * pairs_per_vector(dtype) * 613
    ar = VirtualAllreduce(world, n, dtype, algo, slots=slots, pull=pull, op=op)
    try:
        for launch, kind in enumerate(KINDS):
            vas = make_inputs(world, n, dtype, seed=1000 + 17 * launch, kind=kind, garbage_padding=False)
            ar.load([unpack_loc(_u8(v), dtype) for v in vas])
            for app in ar.ranks:
                app.vc.tensor(torch.uint8).fill_(0xFF)
            torch.cuda.synchronize(DEV)
            ar.run_once()
            want = allreduce_expected(op, vas, dtype)
            for r, (vals, idx) in enumerate(ar.results()):                # synchronizes: status words OK
                got = _bytes(pack_loc(vals, idx, dtype))
                assert mismatches(got, want, dtype) == 0, f"{kind}, rank {r}: {describe(got, want, dtype)}"
    finally:
        ar.close()


@pytest.mark.parametrize("phases", ["reduce_scatter", "all_gather"])
@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_rsag_phases(native, op, dtype, phases):
    """Each phase of ring-rsag on its own: reduce-scatter leaves rank s's own segment reduced, all-gather copies VA's
    segment s of rank s everywhere (bytes untouched, op ignored)."""
    world, esz = 4, pair_bytes(dtype)
    seg = pairs_per_vector(dtype) * 701
    n = seg * world
    ranks = _Ranks(world, extra_words=4096)
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric(n * esz)
        slots = ranks.symmetric(seg * (world - 1) * esz)
        vas = make_inputs(world, n, dtype, seed=77, kind="special")
        for r in range(world):
            va[r].tensor(torch.uint8).copy_(_u8(vas[r]))
            vc[r].tensor(torch.uint8).fill_(0xFF)
            slots[r].tensor(torch.uint8).fill_(0xFF)
        torch.cuda.synchronize(DEV)
        for r in range(world):
            p = ranks.pads[r]
            with torch.cuda.stream(ranks.streams[r]):
                native.ring_rsag(va=va[r].local_ptr, vc=vc[r].local_ptr, slots_local=slots[r].local_ptr,
                                 slots_right=slots[r].ptrs[(r + 1) % world], vc_right=vc[r].ptrs[(r + 1) % world],
                                 arrived_local=p.chunk_word(r), arrived_right=p.chunk_word((r + 1) % world), rank=r,
                                 world=world, n=n, timeout_ns=p.timeout_ns, status=p.status_ptr, dtype=dtype,
                                 ctas=max(1, native.sm_count(DEV) // world), device=DEV,
                                 stream=ranks.streams[r].cuda_stream, phases=phases, op=op)
        for st in ranks.streams:
            st.synchronize()
        assert [native.read_u32(q.status_ptr) for q in ranks.pads] == [native.STATUS_OK] * world
        full = allreduce_expected(op, vas, dtype)
        b = seg * esz
        for r in range(world):
            got = vc[r].tensor(torch.uint8).cpu().numpy().tobytes()
            if phases == "reduce_scatter":
                assert got[r * b:(r + 1) * b] == full[r * b:(r + 1) * b], f"rank {r}"
            else:
                for s in range(world):
                    assert got[s * b:(s + 1) * b] == vas[s][s * b:(s + 1) * b], f"rank {r}, segment {s}"
    finally:
        ranks.close()


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("op", LOC_OPS)
def test_combine(native, op, dtype):
    """VC = op(VC, VA) (ring-unfused's step and ``accumulate``) over whole vectors and, for the 8-byte pairs, an odd
    count whose last vector is half full; nothing after the n pairs is written."""
    L = pairs_per_vector(dtype)
    for i, n in enumerate((L * 3000 + L - 1, 1, L * 777)):
        vc0, va = make_inputs(2, n + GUARD, dtype, seed=600 + i, kind=KINDS[i % len(KINDS)])
        vc = _u8(vc0).to(f"cuda:{DEV}")
        va_d = _u8(va).to(f"cuda:{DEV}")
        native.accumulate(va_d.data_ptr(), vc.data_ptr(), n, dtype, torch.cuda.current_stream(DEV).cuda_stream, op=op)
        torch.cuda.synchronize(DEV)
        got = vc.cpu().numpy().tobytes()
        s = pair_bytes(dtype)
        want = combine_expected(op, vc0[:n * s], va[:n * s], dtype)
        assert mismatches(got[:n * s], want, dtype) == 0, f"n={n}: {describe(got[:n * s], want, dtype)}"
        assert got[n * s:] == vc0[n * s:], f"n={n}: pairs after n were written"
        assert va_d.cpu().numpy().tobytes() == va


@pytest.mark.parametrize("dtype", PAIR_TYPES)
def test_init_and_count_pair(native, dtype):
    from hpc_patterns_b200.ops.allreduce import pack_loc

    n, s = 1001, pair_bytes(dtype)
    v = torch.full((n * s + 64,), 0xAB, dtype=torch.uint8, device=f"cuda:{DEV}")
    st = torch.cuda.current_stream(DEV).cuda_stream
    native.init_pair(v.data_ptr(), n, -3.0, -7, dtype, st)
    torch.cuda.synchronize(DEV)
    want = pack_loc(torch.full((n,), -3.0), torch.full((n,), -7), dtype)
    assert torch.equal(v[:n * s].cpu(), want) and bool((v[n * s:] == 0xAB).all())
    v[s * 500 + s - 1] ^= 1                                      # one padding or index byte of pair 500
    count = torch.zeros(1, dtype=torch.int64, device=f"cuda:{DEV}")
    native.count_pair_mismatch(v.data_ptr(), n, -3.0, -7, dtype, count.data_ptr(), st)
    torch.cuda.synchronize(DEV)
    assert int(count.item()) == 1


# --------------------------------------------------------------- refusals ----
@pytest.mark.parametrize("dtype,op,msg", [
    ("float_int", "sum", "op must be maxloc or minloc for float_int: sum reduces arithmetic types only"),
    ("double_int", "max", "op must be maxloc or minloc for double_int: max reduces arithmetic types only"),
    ("2int", "band", "op must be maxloc or minloc for 2int: band reduces arithmetic types only"),
    ("float", "maxloc", "op must be sum, prod, min or max for float: maxloc reduces value-index pair types only"),
    ("int", "minloc", "op must be sum, prod, min, max, band, bor, bxor, land, lor or lxor for int: minloc reduces "
                      "value-index pair types only"),
])
def test_every_binding_refuses(native, dtype, op, msg):
    world, esz = 2, 16
    n = 64 * world
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
        with pytest.raises(Exception, match=msg):             # the all-gather phase ignores the op, but not these
            native.ring_rsag(va=va[0].local_ptr, vc=vc[0].local_ptr, slots_local=slots[0].local_ptr,
                             slots_right=slots[0].ptrs[1], vc_right=vc[0].ptrs[1], arrived_local=p.chunk_word(0),
                             arrived_right=p.chunk_word(1), rank=0, world=world, n=n, timeout_ns=p.timeout_ns,
                             status=p.status_ptr, dtype=dtype, ctas=1, device=DEV, stream=st, phases="all_gather",
                             op=op)
        with pytest.raises(Exception, match=msg):
            native.allreduce_two_shot(va[0].ptrs, vc[0].ptrs, p.buf.ptrs, p.ticket_ptr, 0, 0, n, 1, p.timeout_ns,
                                      p.status_ptr, dtype, 1, DEV, st, op=op)
        with pytest.raises(Exception, match=msg):
            native.accumulate(va[0].local_ptr, vc[0].local_ptr, n, dtype, st, op=op)
        with pytest.raises(Exception, match="nvls"):
            native.allreduce_nvls(va[0].local_ptr, vc[0].local_ptr, p.buf.ptrs, p.ticket_ptr, 0, 0, n, 1,
                                  p.timeout_ns, p.status_ptr, dtype, 1, DEV, st, op=op)
        torch.cuda.synchronize(DEV)
        assert [native.read_u32(q.status_ptr) for q in ranks.pads] == [native.STATUS_OK] * world
    finally:
        ranks.close()


@pytest.mark.parametrize("op", LOC_OPS)
@pytest.mark.parametrize("dtype", PAIR_TYPES)
def test_virtual_allreduce_constant_check(native, op, dtype):
    """initialize()'s constant data and mismatches()' exact check pass on every rank."""
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    ar = VirtualAllreduce(4, 4 * 2 * 1000, dtype, "ring", op=op)
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


@pytest.mark.parametrize("dtype", PAIR_TYPES)
@pytest.mark.parametrize("args", [["-a"], ["--algo", "ring"], ["--algo", "ring-rsag", "--op", "minloc"]],
                         ids=["a", "ring", "rsag-minloc"])
def test_cli(bin_dir, dtype, args, tmp_path):
    import json

    rows = tmp_path / "rows.jsonl"
    p = _cli([os.path.join(bin_dir, "allreduce." + dtype), "-n", "4", "-p", "18", "--iters", "2", "--json",
              str(rows)] + args)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == 4, p.stdout
    row = json.loads(rows.read_text().splitlines()[-1])
    assert row["op"] == ("minloc" if "minloc" in args else "maxloc") and row["type"] == dtype
    assert row["mismatches"] == 0


@pytest.mark.parametrize("args", [["--type", "float_int", "-S", "--algo", "ring-unfused", "--op", "minloc"],
                                  ["--type", "double_int", "-R", "--slots", "2", "--pull"],
                                  ["--type", "short_int", "-H", "-a"]], ids=["S-unfused", "R-pull", "H-a"])
def test_cli_memory_kinds(bin_dir, args):
    p = _cli([os.path.join(bin_dir, "allreduce"), "-n", "3", "-p", "16", "--iters", "1"] + args)
    assert p.returncode == 0 and p.stdout.count("Passed") == 3, p.stdout + p.stderr


def test_cli_refusals(bin_dir):
    p = _cli([os.path.join(bin_dir, "allreduce.float_int"), "-n", "2", "-p", "12", "-a", "--coll", "nvls"])
    assert p.returncode != 0 and "sum-only" in p.stderr
    p = _cli([os.path.join(bin_dir, "allreduce.2int"), "-n", "2", "-p", "12", "--op", "sum"])
    assert p.returncode != 0 and "reduces arithmetic types only" in p.stderr and "Passed" not in p.stdout
