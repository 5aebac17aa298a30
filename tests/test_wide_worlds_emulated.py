"""The serial-rank drivers of tests/wide_world.py at 9 and 16 ranks without a GPU, on the emulated device of
tests/wide_world_emu.py, so that the harness is trusted before it runs on an H100 (tests/test_gpu_wide_worlds.py):

* every (type, op) pair the two-shot binding takes, through the two-shot and the reduce-scatter; the pinned float and
  double sum across the main / tail boundary; all-to-all, all-gather and all-to-all-v, push and pull, refusals included;
* planted faults, each reported on exactly the ranks hit: a fold of only the first 8 ranks, an arrival in barrier word
  rank % 8, a rank that never arrives, an all-to-all slot rank - 8, a judge that reads rows 0..7 only, a two-shot main
  / tail boundary at U = 2;
* the oracles' data at 16 ranks still has teeth: exact float data stays exact, the 16-bit "full" bands stay finite and
  still round, and the pinned order differs from the other one in a large share of the elements it is checked on.
"""
import pytest
import torch

import tests.allreduce_oracle as aro
import tests.bitop_oracle as bit
import tests.loc_oracle as loc
import tests.lowp_allreduce_oracle as lowp
import tests.reduce_op_oracle as rop
import tests.reduce_scatter_oracle as rso
import tests.wide_world as ww
from tests.alltoallv_oracle import NEGATIVE, PATTERNS, RECV_CAPACITY, SEND_CAPACITY, counts_for
from tests.wide_world_emu import WideWorldEmuNative, install

CASES = ([(t, op) for t in rop.TYPES for op in ("sum",) + rop.OPS]
         + [(t, op) for t in bit.INT_TYPES for op in bit.BIT_OPS]
         + [(t, op) for t in loc.PAIR_TYPES for op in loc.LOC_OPS])


@pytest.fixture
def emu(monkeypatch):
    e = WideWorldEmuNative()
    install(monkeypatch.setattr, e)
    return e


@pytest.fixture
def serial(emu):
    made = []

    def make(world):
        made.append(ww.SerialRanks(world))
        return made[-1]

    yield make
    for sr in made:
        sr.close()


def test_every_pair_the_binding_takes():
    assert len(CASES) == 96 and len(set(CASES)) == 96


# ------------------------------------------------------------------------------------------------ drivers pass ----
@pytest.mark.parametrize("world", [9, 16])
def test_two_shot_and_reduce_scatter_every_pair(serial, world):
    sr = serial(world)
    for dtype, op in CASES:
        ww.two_shot(sr, dtype, op, 1)
        ww.reduce_scatter(sr, dtype, op, 1)


@pytest.mark.parametrize("slice_vec", [37, 512, 3 * 512 + 1])
@pytest.mark.parametrize("world", [9, 16])
@pytest.mark.parametrize("dtype,op", [("float", "sum"), ("double", "sum"), ("half", "sum"), ("int", "sum"),
                                      ("bfloat16", "prod")])
def test_two_shot_across_the_block_boundary(serial, dtype, op, world, slice_vec):
    ww.two_shot(serial(world), dtype, op, slice_vec)


@pytest.mark.parametrize("world", [9, 16])
def test_reduce_scatter_blocks_and_tail(serial, world):
    for dtype, op in (("float", "sum"), ("half", "sum"), ("ulong", "lxor"), ("double", "max")):
        ww.reduce_scatter(serial(world), dtype, op, 4 * 512 + 37)


@pytest.mark.parametrize("pull", [False, True], ids=["push", "pull"])
@pytest.mark.parametrize("world", [9, 16])
def test_all_to_all_and_all_gather(serial, world, pull):
    sr = serial(world)
    for block in (16, 48, 4096 + 16):
        ww.all_to_all(sr, block, pull)
        ww.all_gather(sr, block, pull)


@pytest.mark.parametrize("pull", [False, True], ids=["push", "pull"])
@pytest.mark.parametrize("world", [9, 16])
def test_all_to_all_v_patterns_and_refusals(serial, world, pull):
    v = ww.AllToAllV(serial(world), 48, pull)
    gen = torch.Generator().manual_seed(world)
    for launch, pattern in enumerate(PATTERNS):
        v.launch(counts_for(pattern, world, ww.MEAN, v.cap, launch, gen), launch)
    for rule in (NEGATIVE, SEND_CAPACITY, RECV_CAPACITY):
        v.launch(v.refused(rule), 0)
        v.launch(counts_for("random", world, ww.MEAN, v.cap, rule, gen), 1)


# ----------------------------------------------------------------------------------------------- planted faults ----
def _all(P):
    return list(range(P))


FAULTS = [  # (fault, faulty rank, driver, ranks reported at 16 ranks)
    ("first-8", 12, lambda sr: ww.two_shot(sr, "float", "sum", 3 * 512 + 1), [12]),
    ("first-8", 12, lambda sr: ww.two_shot(sr, "uint", "bor", 1), [12]),
    ("first-8", 9, lambda sr: ww.reduce_scatter(sr, "half", "sum", 4 * 512 + 37), [9]),
    ("first-8", 15, lambda sr: ww.reduce_scatter(sr, "2int", "maxloc", 1), [15]),
    ("word-mod-8", 12, lambda sr: ww.two_shot(sr, "int", "sum", 1), [12]),
    ("word-mod-8", 12, lambda sr: ww.all_gather(sr, 48, True), [12]),
    ("never-arrives", 15, lambda sr: ww.reduce_scatter(sr, "float", "min", 1), [15]),
    ("never-arrives", 15, lambda sr: ww.all_to_all(sr, 16, False), [15]),
    ("slot-minus-8", 9, lambda sr: ww.all_to_all(sr, 48, False), _all(16)),     # rank 9 stores into every rank
    ("slot-minus-8", 9, lambda sr: ww.all_to_all(sr, 48, True), [9]),           # rank 9 loads into its own buffer
    ("rows-below-8", 12, lambda sr: _refused_once(sr, True), [12]),
    ("boundary-u2", 5, lambda sr: ww.two_shot(sr, "float", "sum", 3 * 512 + 1), [5]),
    ("boundary-u2", 5, lambda sr: ww.two_shot(sr, "double", "sum", 512 + 7), [5]),
]


def _refused_once(sr, pull):
    """A negative count in row 12: a judge that reads rows 0..7 only accepts it (pull: only the judge's rank moves)."""
    v = ww.AllToAllV(sr, 48, pull)
    m = v.refused(NEGATIVE)
    m[-1][3], m[12][5] = ww.MEAN // 2, -1
    v.launch(m, 0)


@pytest.mark.parametrize("fault,rank,driver,hit", FAULTS, ids=[f"{f}-{i}" for i, (f, *_) in enumerate(FAULTS)])
def test_planted_faults_are_reported_on_the_ranks_hit(emu, serial, fault, rank, driver, hit):
    sr = serial(16)
    emu.fault, emu.fault_rank = fault, rank
    with pytest.raises(ww.WideWorldError) as e:
        driver(sr)
    assert e.value.ranks == hit, str(e.value)
    if fault == "slot-minus-8" and len(hit) > 1:
        assert "block 9 (from rank 9)" in str(e.value) and "block 1 (from rank 1)" in str(e.value)
    emu.fault = None


def test_the_boundary_fault_is_invisible_where_the_kernels_agree(emu, serial):
    """U = 2 instead of 1 moves no boundary in a slice of fewer than 512 vectors or of a multiple of 1024, and none
    matters to an op whose tail also goes owner first: there the harness must report nothing."""
    sr = serial(16)
    emu.fault, emu.fault_rank = "boundary-u2", 5
    for slice_vec in (511, 2048):
        ww.two_shot(sr, "float", "sum", slice_vec)
    ww.two_shot(sr, "float", "max", 3 * 512 + 1)


def test_a_barrier_that_is_not_armed_is_a_timeout(emu, serial):
    sr = serial(9)
    sr.arm = lambda epoch: None
    with pytest.raises(ww.WideWorldError, match="status word TIMEOUT") as e:
        ww.all_gather(sr, 16, False)
    assert e.value.ranks == list(range(8))          # the last rank finds every word of its epoch


# ---------------------------------------------------------------------------------------- the data at 16 ranks ----
def test_exact_float_data_stays_exact_at_16_ranks():
    """Every partial sum of 16 values in +-EXACT_RANGE lies within +-2^24, where every integer is a float: the edge."""
    assert aro.MAX_RANKS * aro.EXACT_RANGE == 1 << 24
    vas = aro.make_inputs(16, 1 << 14, "float", seed=5, exact=True)
    for v in vas:                                   # the edge itself is in the data
        v[:8] = aro.EXACT_RANGE
    acc = torch.zeros(1 << 14, dtype=torch.float64)
    for k in range(16):
        acc += vas[k].double()
        assert torch.equal(acc.float().double(), acc)
    assert float(acc.abs().max()) == 1 << 24
    assert torch.equal(aro.ring_expected(vas, 5).double(), acc)


@pytest.mark.parametrize("dtype", lowp.LOWP)
def test_lowp_full_bands_stay_finite_and_round_at_16_ranks(dtype):
    """The "full" bands were sized for 8 ranks: at 16 every partial sum, in the 16-bit type (rings) or in fp32
    (two-shot), must stay finite, and the sums must still round."""
    e_bits, m_bits, bias = lowp.FORMAT[dtype]
    lo, step, span, jitter = lowp._FULL_BANDS[dtype]
    largest = 2.0 ** ((1 << e_bits) - 2 - bias) * (2 - 2.0 ** -m_bits)
    bound = 16 * 2.0 ** (lo + span + jitter) + 2.0 ** (lowp._CANCEL_E[dtype] + 1)
    assert bound < largest / 1.5                    # room for the rounding of every partial sum
    vas = lowp.make_inputs(16, 1 << 14, dtype, seed=16)
    x = torch.stack([v.double() for v in vas])
    assert float(x.cumsum(0).abs().max()) < bound
    assert bool(torch.isfinite(lowp.two_shot_expected(vas)).all())
    assert all(bool(torch.isfinite(lowp.ring_expected(vas, r)).all()) for r in (0, 7, 15))
    exact = x.sum(0)
    assert float((lowp.round16(exact.numpy(), dtype).double() != exact).double().mean()) > 0.9
    assert float((x.float().sum(0).double() != exact).double().mean()) > 0.25    # fp32 two-shot sums round too


@pytest.mark.parametrize("world", [9, 16])
@pytest.mark.parametrize("dtype", aro.FLOATING)
def test_the_pinned_order_has_teeth(dtype, world):
    """On the data the GPU file checks, owner first and rank 0 first differ in most elements, so the pin decides."""
    for slice_vec in (37, 512):
        per = slice_vec * 16 // rop.elem_bytes(dtype)
        vas = rso.make_inputs(world, per, dtype, "sum", seed=ww._seed(world, slice_vec, 0), launch=0)
        owner = torch.cat([rso.fold([vas[(s + q) % world][s * per:(s + 1) * per] for q in range(world)], "sum", dtype)
                           for s in range(world)])
        rank0 = rso.fold(list(vas), "sum", dtype)                                   # VA[0] + VA[1] + ...
        pinned = aro.two_shot_sum_pinned(vas)
        assert float((owner != rank0).double().mean()) > 0.4
        assert torch.equal(pinned, rank0 if slice_vec < 512 else owner)


def test_the_pinned_order_splits_at_the_kernels_boundary():
    vas = aro.make_inputs(16, 16 * (512 + 37) * 4, "float", seed=9)
    pinned = aro.two_shot_sum_pinned(vas)
    per = (512 + 37) * 4
    for s in (0, 15):
        head = rso.fold([vas[(s + q) % 16][s * per:s * per + 2048] for q in range(16)], "sum", "float")
        tail = rso.fold([v[s * per + 2048:(s + 1) * per] for v in vas], "sum", "float")
        assert torch.equal(pinned[s * per:(s + 1) * per], torch.cat([head, tail]))
    assert aro.two_shot_u(9) == aro.two_shot_u(16) == 1 and aro.two_shot_u(8) == 2 and aro.two_shot_u(2) == 4
