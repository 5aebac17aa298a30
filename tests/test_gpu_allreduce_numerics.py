"""Element-wise numerics of the allreduce kernels (csrc/kernels/ring_allreduce.cu) on virtual ranks of one GPU.

The miniapps keep the reference's own check (rank r holds r, every element of VC must equal P(P-1)/2), which cannot see
positional errors, stale slots, lane-width errors or the summation order.  Here every rank holds different data per
element and per launch (tests/allreduce_oracle.py), and the kernels are called directly on LocalGroup buffers, so the
sizes, chunk lengths, grids and guards are free:

* the fused ring (push and pull, world-1 slots or two slots with per-chunk acks) must reproduce ``ring_expected`` bit
  for bit: rank r adds VA[r], VA[r-1], ... in that order, in the element type;
* two-shot must give every rank the same bits, equal to the sum for exact data and within the recursive-summation bound
  for random floats (its order is owner-first in the main blocks, rank-0-first in the tail loop);
* VA and 64 guard elements after every VC stay untouched, receive slots start as a NaN / all-ones sentinel, and every
  status word stays OK (a protocol error ends as a timeout status, not a hang).

Each case runs three launches with new data, the epochs (ring) or tickets and barrier epochs (two-shot) advancing as the
miniapp advances them; the host synchronises every stream between launches, standing in for the cross-rank barrier.
``test_virtual_allreduce_plumbing`` runs the same checks through ``AllreduceMiniapp.run_once`` (``VirtualAllreduce``).
"""
import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.allreduce_oracle import (DTYPES, TORCH_DTYPE, describe, elem_bytes, lanes, make_inputs, mismatches,
                                    ring_expected, two_shot_problems)

pytestmark = pytest.mark.gpu

DEV = 0
LAUNCHES = 3
GUARD = 64                  # elements after every VC that no kernel may write
TIMEOUT_S = 10.0
CHUNK_VEC = 8192            # the ring's default chunk: 128 KiB = 8192 16-byte vectors for every element type
RING_VARIANTS = {"push": (0, False), "push-2slots": (2, False), "pull": (0, True), "pull-2slots": (2, True)}


def _max_ctas(world):
    """CTAs per rank that keep every rank's grid co-resident (the ring's CTAs spin on their neighbours)."""
    return max(1, torch.cuda.get_device_properties(DEV).multi_processor_count // world)


class _Ranks:
    """``world`` virtual ranks on one GPU: one stream each, signal pads and symmetric buffers of a LocalGroup."""

    def __init__(self, world, extra_words=0):
        from hpc_patterns_b200.parallel.local import LocalGroup

        self.world = world
        self.group = LocalGroup(world, [DEV] * world)
        self.pads = self.group.pads(extra_words=extra_words, timeout_s=TIMEOUT_S)
        self.buffers = []
        self.streams = [torch.cuda.Stream(DEV) for _ in range(world)]

    def symmetric(self, nbytes, zero=True):
        b = self.group.symmetric(nbytes, zero)
        self.buffers.append(b)
        return b

    def synchronize(self, native):
        for st in self.streams:
            st.synchronize()
        status = [native.read_u32(p.status_ptr) for p in self.pads]
        assert status == [native.STATUS_OK] * self.world, f"status words {status}"

    def close(self):
        torch.cuda.synchronize(DEV)
        for b in self.buffers:
            for x in b:
                x.close()
        for p in self.pads:
            p.close()


def _guard(dtype):
    return make_inputs(1, GUARD, dtype, seed=0xC0FFEE)[0]


def _check_untouched(va, vas, vc, n, guard, td, rank):
    assert mismatches(va.tensor(td).cpu(), vas[rank].cpu()) == 0, f"rank {rank}: VA changed"
    assert mismatches(vc.tensor(td)[n:].cpu(), guard) == 0, f"rank {rank}: a guard after VC was written"


def run_ring(native, world, dtype, variant, nvec, chunk_vec=0, ctas=0, data_device="cpu"):
    """Three launches of the fused ring on ``world`` virtual ranks; every VC must equal ring_expected bit for bit."""
    n_slots, pull = RING_VARIANTS[variant]
    td, L, esz = TORCH_DTYPE[dtype], lanes(dtype), elem_bytes(dtype)
    n, chunk_elems = nvec * L, chunk_vec * L
    n_chunks = native.ring_num_chunks(n, chunk_elems, esz)
    ctas = ctas or _max_ctas(world)
    ranks = _Ranks(world, extra_words=2 * n_chunks)        # arrival words, then ack words
    try:
        va = ranks.symmetric(n * esz)
        vc = ranks.symmetric((n + GUARD) * esz, zero=False)
        slots = ranks.symmetric((2 if n_slots == 2 else max(world - 1, 1)) * n * esz, zero=False)
        guard = _guard(dtype)
        for r in range(world):
            slots[r].tensor().fill_(0xFF)                   # NaN / all-ones: a slot read before it is written shows
            vc[r].tensor(td)[n:].copy_(guard)
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=100 * world + launch, device=data_device)
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
                got, want = vc[r].tensor(td)[:n].to(data_device), ring_expected(vas, r)
                assert mismatches(got, want) == 0, \
                    f"launch {launch}, rank {r}: {mismatches(got, want)} wrong elements, {describe(got, want, L)}"
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("world", range(1, 9))
def test_ring_float_every_world(native, world, variant):
    """1-8 ranks, three full chunks and one vector: acks run in push-2slots from 4 ranks, in pull-2slots from 5."""
    run_ring(native, world, "float", variant, 3 * CHUNK_VEC + 1)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_ring_every_dtype(native, dtype, variant):
    """Every reference type at 5 ranks (acks active in both two-slot variants), full-range integers: a wrong addition
    class (16-bit lanes added as bytes, 64-bit lanes as 32-bit) or a lost carry changes the bits.  The last chunk is
    513 vectors, fewer than the unrolled body needs: only the remainder loop runs there."""
    run_ring(native, 5, dtype, variant, 5 * CHUNK_VEC + 513)


@pytest.mark.parametrize("variant", RING_VARIANTS)
@pytest.mark.parametrize("ctas", ["1", "3", "max"])
@pytest.mark.parametrize("nvec,chunk_vec", [(1, 0), (CHUNK_VEC, 0), (1003, 1), (3 * 2049 + 7, 2049)],
                         ids=["one-vector", "one-chunk", "vector-chunks", "body+remainder-chunks"])
def test_ring_sizes_chunks_and_grids(native, nvec, chunk_vec, ctas, variant):
    """Edges of the chunk loop at 5 ranks: one vector; exactly one default chunk; one vector per chunk (1003 chunks
    dealt round-robin); 2049-vector chunks (unrolled body, then one remainder vector per chunk) -- with one CTA, three
    CTAs and the co-residency maximum per rank."""
    run_ring(native, 5, "float", variant, nvec, chunk_vec, 0 if ctas == "max" else int(ctas))


@pytest.mark.parametrize("variant", RING_VARIANTS)
def test_ring_large_block(native, variant):
    """2^24 + 4 fp32 elements per rank at 5 ranks: 513 default chunks, the last one a single vector.  Data and reference
    stay on the GPU (the reference is still one elementwise IEEE add per hop, in the ring's order)."""
    run_ring(native, 5, "float", variant, (1 << 22) + 1, data_device=f"cuda:{DEV}")


# ---------------------------------------------------------------- two-shot ----
def _block_vec(world):
    """Vectors one CTA reduces per trip of the main loop: 512 threads x U (U = 4 up to 4 ranks, 2 up to 8)."""
    return 512 * (4 if world <= 4 else 2)


def run_two_shot(native, world, dtype, slice_vec, exact, ctas=0):
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
            vas = make_inputs(world, n, dtype, seed=200 * world + launch, exact=exact)
            for r in range(world):
                va[r].tensor(td).copy_(vas[r])
                vc[r].tensor(td)[:n].view(torch.uint8).fill_(0xFF)   # every element must be written by some rank
            torch.cuda.synchronize(DEV)
            for r in range(world):
                p = ranks.pads[r]
                p.barrier_epoch += 1
                grid = native.allreduce_two_shot(va[r].ptrs, vc[r].ptrs, p.buf.ptrs, p.ticket_ptr,
                                                 p.ticket_issued & 0xFFFFFFFF, r, n, p.barrier_epoch, p.timeout_ns,
                                                 p.status_ptr, dtype, ctas, DEV, ranks.streams[r].cuda_stream)
                p.advance_tickets(grid)
            ranks.synchronize(native)
            vcs = [vc[r].tensor(td)[:n].cpu() for r in range(world)]
            problems = two_shot_problems(vcs, vas, exact)
            assert not problems, f"launch {launch}: " + "; ".join(problems)
            for r in range(world):
                _check_untouched(va[r], vas, vc[r], n, guard, td, r)
    finally:
        ranks.close()


SLICES = {"below-one-block": lambda w: 37, "one-block": _block_vec, "blocks+1": lambda w: 3 * _block_vec(w) + 1}


@pytest.mark.parametrize("data", ["exact", "random"])
@pytest.mark.parametrize("slice_", SLICES)
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
def test_two_shot_float(native, world, slice_, data):
    """All three <W,U> instantiations (2/4, 4/4, 8/2) and their ``q < world`` guards; a slice below one block (tail loop
    only), exactly one block (main loop only), k blocks + 1 vector (both)."""
    run_two_shot(native, world, "float", SLICES[slice_](world), data == "exact")


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_shot_every_dtype(native, dtype):
    run_two_shot(native, 5, dtype, 2 * _block_vec(5) + 1, exact=False)


@pytest.mark.parametrize("ctas", [1, 3])
@pytest.mark.parametrize("world", [2, 5, 8])
def test_two_shot_small_grids(native, world, ctas):
    """Fewer CTAs than blocks: each CTA strides over several blocks, then over the tail."""
    run_two_shot(native, world, "float", 5 * _block_vec(world) + 3, exact=False, ctas=ctas)


# ---------------------------------------------------- through the miniapp ----
@pytest.mark.parametrize("dtype", ["float", "int"])
@pytest.mark.parametrize("algo,slots,pull", [("ring", 0, False), ("ring", 2, False), ("ring", 0, True),
                                             ("ring", 2, True), ("twoshot", 0, False), ("ring-unfused", 0, False)],
                         ids=["ring", "ring-2slots", "ring-pull", "ring-pull-2slots", "twoshot", "ring-unfused"])
@pytest.mark.parametrize("world", [4, 5])
def test_virtual_allreduce_plumbing(native, world, algo, slots, pull, dtype):
    """AllreduceMiniapp.run_once on virtual ranks: the argument order of ack / left-neighbour / slot pointers, tickets
    and epochs, with distinct data per rank and per launch.  The unfused ring launches different kernels one after
    the other next to spinning ones, which needs the eager module loading the package asks for when it is imported
    before CUDA starts (this module imports it at collection)."""
    from hpc_patterns_b200.models.allreduce import VirtualAllreduce

    n = world * lanes(dtype) * 5003          # a few default chunks, the last one partial
    ar = VirtualAllreduce(world, n, dtype, algo, slots=slots, pull=pull)
    try:
        for launch in range(LAUNCHES):
            vas = make_inputs(world, n, dtype, seed=300 * world + launch)
            ar.load(vas)
            ar.run_once()
            vcs = ar.results()
            if algo == "twoshot":
                problems = two_shot_problems(vcs, vas, exact=False)
                assert not problems, f"launch {launch}: " + "; ".join(problems)
            else:
                for r in range(world):
                    want = ring_expected(vas, r)
                    assert mismatches(vcs[r], want) == 0, \
                        f"launch {launch}, rank {r}: {describe(vcs[r], want, lanes(dtype))}"
            if algo != "ring-unfused":                  # the unfused ring swaps VA and VB, as the reference does
                for app, v in zip(ar.ranks, vas):
                    assert mismatches(app.va.tensor(v.dtype).cpu(), v) == 0
        assert all(app.launches == LAUNCHES * (1 if algo != "ring-unfused" else 4 * world - 3) for app in ar.ranks)
    finally:
        ar.close()
