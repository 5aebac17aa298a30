"""The allreduce oracle (tests/allreduce_oracle.py) against emulated faulty kernels, on the CPU.

Each fault below is a bug the kernels of csrc/kernels/ring_allreduce.cu could have without the miniapps' constant-value
check noticing.  It is applied to a correct ring (or two-shot) result, and the comparison the GPU tests assert on
(test_gpu_allreduce_numerics.py) must report it on the oracle's data.  Where the constant data of the reference's
check (rank r holds r) hides the fault, that is asserted too: it is the gap the element-wise tests close."""
import numpy as np
import pytest
import torch

from tests.allreduce_oracle import (DTYPES, FLOATING, TORCH_DTYPE, allreduce_bound, lanes, make_inputs, mismatches,
                                    ring_expected, two_shot_problems)

WORLD, RANK = 5, 2
CHUNK_VEC = 64                     # vectors per chunk of the emulated ring
N_VEC = 3 * CHUNK_VEC + 5          # three full chunks and a partial one


def ring_emulated(vas, rank, hop_block=None, add=None):
    """The ring's accumulation with hooks: ``hop_block(t, block)`` edits what hop t reads, ``add`` replaces the add."""
    world = len(vas)
    acc = torch.zeros_like(vas[0])
    for t in range(world):
        src = vas[(rank - t) % world].clone()
        if hop_block is not None:
            src = hop_block(t, src)
        acc = add(acc, src) if add is not None else acc + src
    return acc


def constant_inputs(world, n, dtype):
    """The reference's data: rank r holds r everywhere."""
    return [torch.full((n,), r, dtype=TORCH_DTYPE[dtype]) for r in range(world)]


def _chunk(dtype, c):
    ce = CHUNK_VEC * lanes(dtype)
    return slice(c * ce, (c + 1) * ce)


# ---- the emulated faults: (dtype, fault(vas, rank, other_launch) -> faulty VC, hidden by constant data?) ----------
def shifted_chunk(vas, rank, prev):
    """Hop 2 reads chunk 1 one 16-byte vector too far (a wrong base or stride inside one chunk)."""
    s, v = _chunk("float", 1), lanes("float")

    def hop(t, b):
        if t == 2:
            b[s] = b[s.start + v:s.stop + v].clone()
        return b
    return ring_emulated(vas, rank, hop)


def dropped_tail_chunk(vas, rank, prev):
    """The last, partial chunk is never received (a chunk count rounded down)."""
    tail = 3 * CHUNK_VEC * lanes("float")

    def hop(t, b):
        if t > 0:
            b[tail:] = 0
        return b
    return ring_emulated(vas, rank, hop)


def missing_ack(vas, rank, prev):
    """Two slots without the ack: hop 3 reads chunk 0 of its slot before the sender overwrote it, i.e. hop 1's data."""
    s, world = _chunk("float", 0), len(vas)

    def hop(t, b):
        if t == 3:
            b[s] = vas[(rank - (t - 2)) % world][s]
        return b
    return ring_emulated(vas, rank, hop)


def stale_launch(vas, rank, prev):
    """An arrival word of the previous launch satisfies a wait: hop 2 reads chunk 2 of the previous launch's data."""
    s, world = _chunk("float", 2), len(vas)

    def hop(t, b):
        if t == 2:
            b[s] = prev[(rank - t) % world][s]
        return b
    return ring_emulated(vas, rank, hop)


def long_add_without_carry(vas, rank, prev):
    """A 64-bit add done as two 32-bit adds with no carry from the low half into the high half."""
    lo = 0xFFFFFFFF

    def add(a, b):
        return (((a >> 32) + (b >> 32)) << 32) | (((a & lo) + (b & lo)) & lo)
    return ring_emulated(vas, rank, add=add)


def short_as_bytes(vas, rank, prev):
    """16-bit lanes added with the 8-bit class (__vadd4 instead of __vadd2): no carry between the two bytes."""
    def add(a, b):
        return (a.view(torch.uint8) + b.view(torch.uint8)).view(a.dtype)
    return ring_emulated(vas, rank, add=add)


def swapped_f64_lanes(vas, rank, prev):
    """Hop 1 swaps the two f64 lanes of one 16-byte vector (lo/hi halves of the uint4 mixed up)."""
    def hop(t, b):
        if t == 1:
            pair = b.view(-1, 2)
            pair[7] = pair[7].flip(0).clone()
        return b
    return ring_emulated(vas, rank, hop)


FAULTS = [("float", shifted_chunk, True), ("float", dropped_tail_chunk, False), ("float", missing_ack, False),
          ("float", stale_launch, True), ("long", long_add_without_carry, True), ("ulong", long_add_without_carry, True),
          ("short", short_as_bytes, True), ("ushort", short_as_bytes, True), ("double", swapped_f64_lanes, True)]


@pytest.mark.parametrize("dtype,fault,hidden", FAULTS, ids=[f"{f.__name__}-{d}" for d, f, _ in FAULTS])
def test_emulated_ring_fault_is_reported(dtype, fault, hidden):
    n = N_VEC * lanes(dtype)
    vas = make_inputs(WORLD, n, dtype, seed=11)
    prev = make_inputs(WORLD, n, dtype, seed=10)
    for rank in range(WORLD):
        want = ring_expected(vas, rank)
        assert mismatches(ring_emulated(vas, rank), want) == 0
        assert mismatches(fault(vas, rank, prev), want) > 0, f"{fault.__name__} not reported at rank {rank}"
    const = constant_inputs(WORLD, n, dtype)
    missed = mismatches(fault(const, RANK, const), ring_expected(const, RANK)) == 0
    assert missed == hidden


def test_two_shot_rank_disagreement_is_reported():
    """One element of one rank's VC one ulp off: within the summation bound, but not bit-identical to rank 0."""
    vas = make_inputs(WORLD, N_VEC * 4, "float", seed=3)
    vcs = [ring_expected(vas, 0) for _ in range(WORLD)]
    assert two_shot_problems(vcs, vas, exact=False) == []
    vcs[3] = vcs[3].clone()
    vcs[3][77] = torch.nextafter(vcs[3][77], torch.tensor(float("inf")))
    problems = two_shot_problems(vcs, vas, exact=False)
    assert len(problems) == 1 and problems[0].startswith("rank 3 differs")


@pytest.mark.parametrize("dtype", FLOATING)
def test_two_shot_bound_accepts_every_order_and_rejects_a_wrong_sum(dtype):
    """Sums in the owner-first order of the main blocks and the rank-0-first order of the tail loop both pass the
    bound; a lost addend does not, nor does a NaN; exact data must match bit for bit."""
    vas = make_inputs(8, 4096, dtype, seed=5)
    for rank in range(8):
        rot = vas[rank:] + vas[:rank]
        owner_first = ring_expected(rot[::-1], 7)     # rot[0] + rot[1] + ... + rot[7]
        assert two_shot_problems([owner_first] * 8, vas, exact=False) == []
    ref, bound = allreduce_bound(vas)
    assert bool((bound > 0).all()) and bool((bound < 1e-4 * ref.abs().max()).all())
    wrong = ring_expected(vas[:-1], 0)
    assert two_shot_problems([wrong] * 8, vas, exact=False)
    nan = ring_expected(vas, 0).clone()
    nan[5] = float("nan")
    assert two_shot_problems([nan] * 8, vas, exact=False)
    ex = make_inputs(8, 4096, dtype, seed=5, exact=True)
    good = ring_expected(ex, 3)
    assert two_shot_problems([good] * 8, ex, exact=True) == []
    off = good.clone()
    off[9] += 1
    assert two_shot_problems([off] * 8, ex, exact=True)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ring_expected_matches_a_numpy_loop(dtype):
    np_type = {"float": np.float32, "int": np.int32, "uint": np.uint32, "double": np.float64, "long": np.int64,
               "ulong": np.uint64, "short": np.int16, "ushort": np.uint16, "uchar": np.uint8}[dtype]
    for world in (1, 3, 5):
        vas = make_inputs(world, 1000 * lanes(dtype), dtype, seed=world)
        arrays = [v.numpy().view(np_type) for v in vas]
        for rank in range(world):
            acc = np.zeros_like(arrays[0])
            for t in range(world):
                acc = acc + arrays[(rank - t) % world]      # numpy wraps integer arrays modulo 2^bits
            assert ring_expected(vas, rank).numpy().tobytes() == acc.tobytes()


@pytest.mark.parametrize("dtype", DTYPES)
def test_inputs_differ_per_rank_element_and_seed(dtype):
    n = 4096 * lanes(dtype)
    a, b = make_inputs(3, n, dtype, seed=1), make_inputs(3, n, dtype, seed=2)
    assert mismatches(a[0], make_inputs(3, n, dtype, seed=1)[0]) == 0        # reproducible
    assert mismatches(a[0], a[1]) > n // 2 and mismatches(a[0], b[0]) > n // 2
    assert len(torch.unique(a[0])) > min(n // 4, 200)
    if dtype not in FLOATING:
        # full range: sums wrap, and the low bytes of two ranks carry into the next byte for many elements
        info = torch.iinfo(a[0].dtype)
        quarter = (info.max - info.min) // 4
        assert int(a[0].min()) < info.min + quarter and int(a[0].max()) > info.max - quarter
        carry = (a[0].view(torch.uint8).int() + a[1].view(torch.uint8).int()) > 255
        assert int(carry.sum()) > carry.numel() // 4


@pytest.mark.parametrize("dtype", FLOATING)
def test_exact_floats_sum_exactly_in_every_order(dtype):
    vas = make_inputs(8, 1 << 14, dtype, seed=9, exact=True)
    assert all(bool((v.abs() <= 1 << 20).all()) and bool((v == v.round()).all()) for v in vas)
    ref, _ = allreduce_bound(vas)
    for rank in range(8):
        assert torch.equal(ring_expected(vas, rank).to(torch.float64), ref)
