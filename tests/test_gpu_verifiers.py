"""The on-device checks against planted faults: every case puts a field on the device, counts the wrong elements on the
host under the check's own rule (tests/field_compare.py) and asserts that the kernel reports exactly that number.

Covered: ``halo_verify_from_init`` and ``halo_verify_step`` for every field type, ``verify_triad``, ``verify_pattern``
and ``count_mismatch``; then K-halo itself against ``reference_steps`` where the field runs into inf and NaN or through
subnormals into ±0.  Positions: element 0, the last element of the last row, every lane of a 16-byte vector, the first
and last row of a slab, the second and third grid-stride pass, 32 faults in one warp, one fault in every CTA, and a
field where every element is wrong.
"""
import numpy as np
import pytest
import torch

from hpc_patterns_b200.models.halo import DTYPES, VirtualRing, initial_field, reference_steps
from hpc_patterns_b200.ops.halo import stencil_step_reference
from tests.field_compare import count_far, count_wrong
from tests.verifier_faults import (TYPES, assert_run_reaches, bits_of, lanes, other_nan, run_field, special_counts,
                                   special_step, ulp_away, value_row)

pytestmark = pytest.mark.gpu

SMS = 132
INIT_CTAS, INIT_THREADS = SMS * 16, 128     # launch_halo_verify_from_init: one column per thread
STEP_CTAS, STEP_THREADS = SMS * 8, 256      # launch_halo_verify_step: one 16-byte vector per thread
PASS = INIT_CTAS * INIT_THREADS             # 270 336 columns (or vectors) per grid-stride pass of both
assert PASS == STEP_CTAS * STEP_THREADS
IDS = {t: DTYPES[t] for t in TYPES}


@pytest.fixture(scope="module", autouse=True)
def dev():
    torch.cuda.set_device(0)
    assert torch.cuda.get_device_properties(0).multi_processor_count == SMS, "the grid caps assume an H100 SXM"
    return torch.device("cuda", 0)


def _st():
    return torch.cuda.current_stream().cuda_stream


def verify_init(native, u, rank, world, steps, alpha, s):
    rows, n = u.shape
    u = u.cuda().contiguous()
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    native.halo_verify_from_init(u.data_ptr(), rows, n, rank, world, steps, alpha, s, cnt.data_ptr(), _st(),
                                 DTYPES[u.dtype])
    torch.cuda.synchronize()
    return int(cnt.item())


def verify_step(native, new, old, up, dn, alpha, s):
    rows, n = old.shape
    new, old, up, dn = (t.cuda().contiguous() for t in (new, old, up, dn))
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    native.halo_verify_step(new.data_ptr(), old.data_ptr(), up.data_ptr(), dn.data_ptr(), rows, n, alpha, s,
                            cnt.data_ptr(), _st(), DTYPES[old.dtype])
    torch.cuda.synchronize()
    return int(cnt.item())


def bump(t, where):
    """+1 ulp (away from zero) at every (row, column) of ``where`` of a host field; returns the number of faults."""
    b = bits_of(t)
    where = sorted(set(where))
    for r, c in where:
        b[r, c] += 1
    return len(where)


def position_table(rows, n, lanes_, threads, ctas):
    """Named fault positions (row, column) in a [rows, n] slab whose columns are checked lanes_ per thread, by a grid of
    ctas x threads with a grid stride (n must span three passes)."""
    per = ctas * threads
    assert n // lanes_ > 2 * per
    return {
        "element 0": [(0, 0)],
        "last element of the last row": [(rows - 1, n - 1)],
        "first row": [(0, 12345)],
        "last row": [(rows - 1, 54321)],
        "every lane of one vector": [(1, 9 * lanes_ + k) for k in range(lanes_)],
        "every lane of the last vector": [(rows - 1, n - lanes_ + k) for k in range(lanes_)],
        "second grid-stride pass": [(1, (per + 5) * lanes_)],
        "third grid-stride pass": [(rows - 1, (2 * per + 77) * lanes_ + lanes_ - 1)],
        "32 faults in one warp": [(1, (4096 + k) * lanes_) for k in range(32)],
        "one warp, every row": [(r, (64 + k) * lanes_ + k % lanes_) for k in range(32) for r in range(rows)],
        "one fault in every CTA": [(c % rows, (c * threads + c % threads) * lanes_ + c % lanes_) for c in range(ctas)],
        "every CTA of the third pass": [(c % rows, (2 * per + c * threads + 31) * lanes_) for c in range(ctas)],
    }


# ------------------------------------------------------------------------------------------------ verify_from_init ----
@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
@pytest.mark.parametrize("run", ["grow", "decay"])
def test_verify_init_special_fields(native, dtype, run):
    """Correct fields with NaN / inf (growing run) and subnormals / ±0 (decaying run) give 0; the value faults that
    only such fields have are each counted once, and a NaN with another payload is not counted."""
    world, rows, n = 2, 13, 4096 + 8
    for cp in (0, 1):
        field, steps, alpha, s = run_field(world, rows, n, dtype, run, cp)
        assert_run_reaches(field, run, cp)
        for rank in range(world):
            want = field[rank * rows:(rank + 1) * rows].contiguous()
            assert verify_init(native, want, rank, world, steps, alpha, s) == 0, (run, cp, rank)
            got, d = want.clone(), want.double()
            planted = []
            if run == "grow":
                nan = torch.nonzero(torch.isnan(d))
                assert len(nan) >= 2
                planted += [(tuple(nan[0].tolist()), torch.tensor(1.0, dtype=dtype), True),
                            (tuple(nan[-1].tolist()), other_nan(dtype), False)]
                inf = torch.nonzero(torch.isinf(d))
                if len(inf):
                    planted.append((tuple(inf[0].tolist()), torch.tensor(torch.finfo(dtype).max, dtype=dtype), True))
            else:
                zero, neg = d == 0, torch.signbit(d)
                for mask, val in ((zero & neg, 0.0), (zero & ~neg, -0.0)):
                    idx = torch.nonzero(mask)
                    if len(idx):
                        planted.append((tuple(idx[len(idx) // 2].tolist()), torch.tensor(val, dtype=dtype), True))
                sub = torch.nonzero((d != 0) & (d.abs() < torch.finfo(dtype).tiny))
                if len(sub):
                    r, c = sub[0].tolist()
                    planted.append(((r, c), torch.tensor(0.0, dtype=dtype) * torch.sign(want[r, c]), True))
            assert planted
            for (r, c), val, _ in planted:
                got[r, c] = val
            expected = sum(counted for _, _, counted in planted)
            assert count_wrong(got, want) == expected
            assert verify_init(native, got, rank, world, steps, alpha, s) == expected, (run, cp, rank, planted)


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_verify_init_positions_and_counting(native, dtype):
    """+1 ulp at every position of the table, each category on its own, and a field where every element is wrong."""
    rows, n, steps = 3, 3 * PASS + 1000, 2
    want = reference_steps(initial_field(1, rows, n, dtype), steps)
    assert verify_init(native, want, 0, 1, steps, 0.5, 0.25) == 0
    for name, where in position_table(rows, n, 1, INIT_THREADS, INIT_CTAS).items():
        got = want.clone()
        expected = bump(got, where)
        assert count_wrong(got, want) == expected
        assert verify_init(native, got, 0, 1, steps, 0.5, 0.25) == expected, name
    got = want.clone()
    bits_of(got).bitwise_xor_(1)
    assert verify_init(native, got, 0, 1, steps, 0.5, 0.25) == rows * n == count_wrong(got, want)


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
@pytest.mark.parametrize("rows,world", [(4, 32), (1, 128), (2, 3)])
def test_verify_init_ranks(native, dtype, rows, world):
    """Rank > 0 compares its own rows of the global field, up to rows * world = 128."""
    n, steps = 2048 + 24, 3
    field = reference_steps(initial_field(world, rows, n, dtype), steps)
    for rank in sorted({1, world // 2, world - 1}):
        want = field[rank * rows:(rank + 1) * rows].contiguous()
        assert verify_init(native, want, rank, world, steps, 0.5, 0.25) == 0, rank
        got = want.clone()
        expected = bump(got, [(0, 0), (rows - 1, n - 1), (rank % rows, 100 + rank)])
        assert verify_init(native, got, rank, world, steps, 0.5, 0.25) == expected, rank
    if world > 1:   # another rank's rows are wrong here
        other = field[0:rows].contiguous()
        assert verify_init(native, other, world - 1, world, steps, 0.5, 0.25) == count_wrong(other, field[-rows:])


@pytest.mark.parametrize("rows,world", [(1, 129), (43, 3), (129, 1)])
def test_verify_init_refuses_more_than_128_global_rows(native, rows, world):
    u = torch.zeros(rows, 64, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    with pytest.raises(Exception, match="128"):
        native.halo_verify_from_init(u.data_ptr(), rows, 64, 0, world, 1, 0.5, 0.25, cnt.data_ptr(), _st(), "float")
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------- verify_step ----
@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_verify_step_value_faults(native, dtype):
    """The value table on a one-row slab whose reference step is the row itself (alpha = s = 1, neighbours all -0)."""
    n = 64 * lanes(dtype)
    want, got, expected, where = value_row(dtype, n)
    old = want[None].contiguous()
    z = torch.full((n,), -0.0, dtype=dtype)
    assert count_wrong(stencil_step_reference(old, z, z, 1.0, 1.0), old) == 0
    assert verify_step(native, old, old, z, z, 1.0, 1.0) == 0
    assert count_wrong(got, want) == expected
    assert verify_step(native, got[None], old, z, z, 1.0, 1.0) == expected
    for name, i in where.items():     # one fault at a time: each is counted (or not) on its own
        one = want.clone()
        one[i] = got[i]
        assert verify_step(native, one[None], old, z, z, 1.0, 1.0) == count_wrong(one, want), name


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
@pytest.mark.parametrize("alpha,s", [(0.5, 0.25), (0.3, 0.7)])
def test_verify_step_special_inputs(native, dtype, alpha, s):
    """A step whose input holds ±0, subnormals, the largest finite values, ±inf and NaN: its exact output (-0, ±inf,
    NaN among it) gives 0, and random bit flips anywhere, NaN positions included, are counted by the rule."""
    rows, n = 5, 2048 * lanes(dtype)
    old, up, dn = special_step(dtype, rows, n)
    want = stencil_step_reference(old, up, dn, alpha, s)
    c = special_counts(want)
    assert c["nan"] and c["inf"] and c["-0"] and c["+0"] and c["subnormal"], c
    assert verify_step(native, want, old, up, dn, alpha, s) == 0
    g = torch.Generator().manual_seed(11)
    got = want.clone()
    idx = torch.randint(0, rows * n, (500,), generator=g)
    bit = torch.randint(0, 8 * want.element_size(), (500,), generator=g)
    flat = bits_of(got).view(-1)
    for i, b in zip(idx.tolist(), bit.tolist()):
        flat[i] ^= torch.tensor(1 << b if b < 8 * want.element_size() - 1 else -(1 << b)).to(flat.dtype)
    expected = count_wrong(got, want)
    assert 0 < expected <= 500
    assert verify_step(native, got, old, up, dn, alpha, s) == expected


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_verify_step_positions_and_counting(native, dtype):
    rows, L = 3, lanes(dtype)
    n = (3 * PASS + 40) * L
    g = torch.Generator().manual_seed(3)
    ext = (torch.randint(-512, 513, (rows + 2, n), generator=g, dtype=torch.int16).float() / 16).to(dtype)
    old, up, dn = ext[1:-1].contiguous(), ext[0].contiguous(), ext[-1].contiguous()
    want = stencil_step_reference(old, up, dn)
    assert verify_step(native, want, old, up, dn, 0.5, 0.25) == 0
    for name, where in position_table(rows, n, L, STEP_THREADS, STEP_CTAS).items():
        got = want.clone()
        expected = bump(got, where)
        assert verify_step(native, got, old, up, dn, 0.5, 0.25) == expected, name
    got = want.clone()
    bits_of(got).bitwise_xor_(1)
    assert verify_step(native, got, old, up, dn, 0.5, 0.25) == rows * n == count_wrong(got, want)


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_verify_step_recomputes_from_neighbour_rows(native, dtype):
    """A changed neighbour row (up, dn) or input row is counted as the output elements it changes: the check
    recomputes the step from the rows it is given, not from the output."""
    rows, n = 4, 1024 * lanes(dtype)
    g = torch.Generator().manual_seed(5)
    ext = (torch.randint(-512, 513, (rows + 2, n), generator=g, dtype=torch.int16).float() / 16).to(dtype)
    old, up, dn = ext[1:-1].contiguous(), ext[0].contiguous(), ext[-1].contiguous()
    new = stencil_step_reference(old, up, dn)
    cols = [0, 7, n // 2, n - 1]
    for which in ("up", "dn", "row 0", "row 2", f"row {rows - 1}"):
        o, u, d = old.clone(), up.clone(), dn.clone()
        target = {"up": u, "dn": d}.get(which)
        if target is None:
            target = o[int(which.split()[1])]
        target[cols] = target[cols] + 7
        expected = count_wrong(new, stencil_step_reference(o, u, d))
        assert expected >= len(cols)
        assert verify_step(native, new, o, u, d, 0.5, 0.25) == expected, which


# ------------------------------------------------------------------------------------------- the other three checks ----
def _spread(n, threads, ctas):
    """Fault indices of a 1-D buffer checked one element per thread: the position table of the halo checks."""
    per = threads * ctas
    return {
        "element 0": [0],
        "last element": [n - 1],
        "32 faults in one warp": list(range(4096, 4128)),
        "one fault in every CTA": [c * threads + c % threads for c in range(ctas)],
        "second grid-stride pass": [per + 5],
        "third grid-stride pass": [2 * per + 77] if n > 2 * per + 77 else [n - 2],
    }


@pytest.mark.parametrize("src_rank", [0, 5])
def test_verify_triad_counts_exactly(native, src_rank):
    from hpc_patterns_b200.ops.fused import triad_inputs_reference

    n = 3 * 270336 + 7                   # launch_verify_triad: 256 x 1056, one element per thread
    b, c = triad_inputs_reference(n, src_rank)
    want = b + 3.0 * c                   # small integers: exact, as the kernel's fmaf
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")

    def run(a):
        a = a.cuda()
        cnt.zero_()
        native.verify_triad(a.data_ptr(), n, src_rank, 3.0, cnt.data_ptr(), _st())
        torch.cuda.synchronize()
        return int(cnt.item())

    assert run(want) == 0
    for name, where in _spread(n, 256, 1056).items():
        got = want.clone()
        got[where] += 1.0
        assert run(got) == len(set(where)), name
    assert run(want + 0.5) == n
    other = triad_inputs_reference(n, src_rank + 1)[0]      # another rank's data
    assert run(other) == int((other != want).sum())
    # Displacement: a block moved by its own size (a tile at its neighbour's offset) and a stale stage of the default
    # TMA ring (6 stages of 16 KiB: tile j holds tile j - 6).  The count must match the host AND cover the moved
    # elements: a payload that repeats every 4 KiB would give 0 on both sides.
    for name, (shift, lo, size) in {"4 KiB block": (1024, 8192, 1024), "16 KiB block": (4096, 16384, 4096),
                                    "64 KiB block": (16384, 65536, 16384),
                                    "stale stage": (6 * 4096, 18 * 4096, 4096)}.items():
        got = want.clone()
        got[lo:lo + size] = want[lo - shift:lo - shift + size]
        host = int((got != want).sum())
        assert run(got) == host >= 0.99 * size, (name, host)


@pytest.mark.parametrize("n_words", [1, 17, 31, 4097, 3 * 135168 + 3])
def test_verify_pattern_counts_exactly_and_sums(native, n_words):
    from hpc_patterns_b200.ops.p2p import pattern_reference

    seed = 0xDEADBEEF
    ref = pattern_reference(n_words, seed)                       # int64 holding uint32 words
    counters = torch.zeros(2, dtype=torch.int64, device="cuda")

    def run(words):
        buf = torch.from_numpy(words.astype(np.uint32).view(np.int32)).cuda()
        counters.zero_()
        native.verify_pattern(buf.data_ptr(), n_words, seed, counters.data_ptr(), counters.data_ptr() + 8)
        torch.cuda.synchronize()
        bad, total = (int(x) for x in counters.cpu())
        assert total & 0xFFFFFFFFFFFFFFFF == int(words.astype(np.uint64).sum(dtype=np.uint64))
        return bad

    words = ref.numpy().astype(np.uint64)
    assert run(words) == 0
    for name, where in _spread(n_words, 256, 528).items():   # launch_verify_pattern: 256 x 528
        where = sorted({i for i in where if i < n_words})
        got = words.copy()
        got[where] ^= 1
        assert run(got) == len(where), name
    assert run(words ^ 0x80000000) == n_words


COUNT_TYPES = {"float": torch.float32, "double": torch.float64, "int": torch.int32, "uint": torch.int32,
               "long": torch.int64, "ulong": torch.int64, "short": torch.int16, "ushort": torch.int16,
               "uchar": torch.uint8, "bfloat16": torch.bfloat16, "half": torch.float16}


@pytest.mark.parametrize("dtype", sorted(COUNT_TYPES))
def test_count_mismatch_counts_exactly(native, dtype):
    """|x - 13| < 1e-6 in double, as the reference checks; NaN counts, a float or double 1 ulp off 13 does not."""
    td = COUNT_TYPES[dtype]
    n = 3 * 270336 + 5                   # launch_count_mismatch: 256 x 1056
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")

    def run(v):
        v = v.cuda()
        cnt.zero_()
        native.count_mismatch(v.data_ptr(), n, 13.0, dtype, cnt.data_ptr(), _st())
        torch.cuda.synchronize()
        return int(cnt.item())

    want = torch.full((n,), 13, dtype=td)
    assert run(want) == 0
    for name, where in _spread(n, 256, 1056).items():
        got = want.clone()
        got[where] = 12
        assert run(got) == len(set(where)), name
    got = want.clone()
    got[[0, n // 3, n - 1]] = 14
    if td.is_floating_point:
        got[[5, 6]] = float("nan")
        up = ulp_away(torch.tensor(13.0, dtype=td))
        got[[7, 8, 2 * n // 3]] = up
        wide = td in (torch.float32, torch.float64)
        expected = 3 + 2 + (0 if wide else 3)        # a 16-bit ulp of 13 is far beyond 1e-6
        if wide:
            assert 0 < float(up) - 13.0 < 1e-6
    else:
        expected = 3
    assert count_far(got.double().numpy(), 13.0) == expected
    assert run(got) == expected
    assert run(torch.zeros(n, dtype=td)) == n


# ---------------------------------------------------------------------------------- K-halo at the special values ----
@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("run", ["grow", "decay"])
def test_khalo_matches_reference_into_inf_nan_and_signed_zeros(native, dtype, world, mode, run):
    """The fused step on virtual ranks, bit for bit (NaN as a class) against reference_steps where the field runs into
    inf and NaN, or through subnormals into ±0; both checks agree on every rank."""
    rows = {1: 26, 2: 13, 3: 9}[world]
    message = 4096 + 48
    n = message // torch.empty(0, dtype=dtype).element_size()
    first, alpha, s = run_field(world, rows, n, dtype, run, 0)[1:]
    second = run_field(world, rows, n, dtype, run, 1)[1]
    ring = VirtualRing(world, message_bytes=message, rows=rows, mode=mode, devices=[0] * world, alpha=alpha, s=s,
                       dtype=dtype)
    try:
        start = initial_field(world, rows, n, dtype)
        ring.step(first)
        for cp, steps in ((0, first), (1, second)):
            if cp == 1:
                ring.step(second - first, persistent=True)
            want = reference_steps(start, steps, alpha, s)
            assert_run_reaches(want, run, cp)
            got = ring.gather()
            assert count_wrong(got, want) == 0, (steps, special_counts(got), special_counts(want))
            for hs in ring.ranks:
                assert hs.verify_from_init() == 0, (steps, hs.rank)
                assert hs.verify_last_step() == 0, (steps, hs.rank)
    finally:
        ring.close()
