"""Executable model of the reduce-scatter + all-gather ring (ring_rsag_kernel, csrc/kernels/ring_allreduce.cu), on the
CPU, plus its oracle and its host-thread twin in bin/allreduce.

The hop rules live in csrc/kernels/ring_order.h (rsag_*) and are called here through the extension, so the model runs
the SAME rules the device code runs.  P ranks x G CTAs are coroutines that a random scheduler interleaves chunk by
chunk; values are symbolic sum trees, so the model sees the order of every add.  It checks, for all three phases:
no slot or VC chunk is read before it is written in this launch, none is written twice (so none is overwritten before
it is read), no rank pushes into its right neighbour's own segment, there is no deadlock, and the result has the
oracle's order.  Each mutation of the rules must be caught.
"""
import os
import random
import subprocess

import numpy as np
import pytest
import torch
from hypothesis import given, settings, strategies as st

import hpc_patterns_b200
from tests.allreduce_oracle import DTYPES, TORCH_DTYPE, make_inputs, mismatches, ring_expected
from tests.rsag_oracle import reduce_scatter_expected, rsag_expected

PHASES = ("allreduce", "reduce_scatter", "all_gather")
MUTATIONS = ("wait_one_early", "forward_own_va", "push_into_right_own_segment", "segment_off_by_one")


class Violation(Exception):
    pass


def _phase_id(C, phase):
    return {"allreduce": C.RSAG_ALLREDUCE, "reduce_scatter": C.RSAG_REDUCE_SCATTER,
            "all_gather": C.RSAG_ALL_GATHER}[phase]


def _reached(seen, want):
    """epoch_reached of csrc/common/signal.cuh: wrap-safe comparison of 32-bit epochs."""
    d = (seen - want) & 0xFFFFFFFF
    return d < 0x80000000


def _expected_sum(world, s, c):
    """((VA[s+1] + VA[s+2]) + ...) + VA[s] of chunk c, as a sum tree (the oracle's order)."""
    acc = ("va", (s + 1) % world, s, c)
    for k in range(2, world + 1):
        acc = (acc, ("va", (s + k) % world, s, c))
    return acc


def run_launch(world, n_chunks, ctas, phase, seed, arrived, epoch_base, mutation=None):
    """One launch of ``phase`` on every rank; ``arrived`` (per rank, per chunk) carries over between launches."""
    C = hpc_patterns_b200.native()
    ph = _phase_id(C, phase)
    rng = random.Random(seed)
    va = [[[("va", r, s, c) for c in range(n_chunks)] for s in range(world)] for r in range(world)]
    vc = [[[None] * n_chunks for _ in range(world)] for _ in range(world)]
    slots = [[[None] * n_chunks for _ in range(max(world - 1, 1))] for _ in range(world)]
    unread = [[[False] * n_chunks for _ in range(max(world - 1, 1))] for _ in range(world)]
    first, last = C.rsag_first_hop(ph, world), C.rsag_last_hop(ph, world)
    work = {(r, g): [(h, c) for h in range(first, last + 1) for c in range(g, n_chunks, ctas)]
            for r in range(world) for g in range(ctas)}
    pos = {k: 0 for k in work}

    def seg_of(h, r):
        s = C.rsag_segment(h, r, world)
        return (s + 1) % world if mutation == "segment_off_by_one" else s

    def runnable(r, h, c):
        if not C.rsag_waits(h, ph, world):
            return True
        want = C.rsag_arrival(h, ph, world) - (1 if mutation == "wait_one_early" else 0)
        return _reached(arrived[r][c], (epoch_base + want) & 0xFFFFFFFF)

    def step(r, h, c):
        right = (r + 1) % world
        s = seg_of(h, r)
        if C.rsag_reads_vc(h, world):
            x = vc[r][s][c]
            if x is None:
                raise Violation(f"rank {r} hop {h} reads VC[{s}] chunk {c} before it was written")
        else:
            x = va[r][s][c]
        own_va = x
        k = C.rsag_src_slot(h, ph, world)
        if k >= 0:
            if not unread[r][k][c]:
                raise Violation(f"rank {r} hop {h} reads slot {k} chunk {c} before it was written")
            unread[r][k][c] = False
            x = (slots[r][k][c], x)
        if C.rsag_writes_own_vc(h, world):
            if vc[r][s][c] is not None:
                raise Violation(f"rank {r} hop {h} overwrites its own VC[{s}] chunk {c}")
            vc[r][s][c] = x
        if C.rsag_forwards(h, ph, world):
            fs = C.rsag_fwd_slot(h, world)
            if fs >= 0:
                if slots[right][fs][c] is not None:
                    raise Violation(f"rank {r} hop {h} overwrites slot {fs} chunk {c} of rank {right}")
                slots[right][fs][c] = own_va if mutation == "forward_own_va" else x
                unread[right][fs][c] = True
            else:
                t = right if mutation == "push_into_right_own_segment" else s
                if t == right:
                    raise Violation(f"rank {r} hop {h} pushes into rank {right}'s own segment")
                if vc[right][t][c] is not None:
                    raise Violation(f"rank {r} hop {h} overwrites VC[{t}] chunk {c} of rank {right}")
                vc[right][t][c] = x
            arrived[right][c] = (epoch_base + C.rsag_arrival(h + 1, ph, world)) & 0xFFFFFFFF

    while True:
        ready = [k for k in work if pos[k] < len(work[k]) and runnable(k[0], *work[k][pos[k]])]
        if not ready:
            break
        k = rng.choice(ready)
        step(k[0], *work[k][pos[k]])
        pos[k] += 1
    stuck = [k for k in work if pos[k] < len(work[k])]
    if stuck:
        raise Violation(f"deadlock: {stuck[:4]} blocked")
    if any(unread[r][k][c] for r in range(world) for k in range(len(unread[r])) for c in range(n_chunks)):
        raise Violation("a slot chunk was written and never read")
    for r in range(world):
        for s in range(world):
            for c in range(n_chunks):
                if phase == "allreduce":
                    want = _expected_sum(world, s, c)
                elif phase == "reduce_scatter":
                    want = _expected_sum(world, s, c) if s == r else None     # only own VC[r] is written
                else:
                    want = ("va", s, s, c)
                if vc[r][s][c] != want:
                    raise Violation(f"rank {r} VC[{s}] chunk {c}: got {vc[r][s][c]}, want {want}")
    return (epoch_base + C.rsag_epoch_advance(ph, world)) & 0xFFFFFFFF


def simulate(world, n_chunks, ctas, phases, seed, epoch_base=0, mutation=None):
    """Consecutive launches (separated by a barrier, as on the device) that share the arrival words."""
    arrived = [[epoch_base] * n_chunks for _ in range(world)]
    base = epoch_base
    for i, phase in enumerate(phases):
        base = run_launch(world, n_chunks, ctas, phase, seed + i, arrived, base, mutation)
    return base


@given(world=st.integers(1, 9), n_chunks=st.integers(1, 5), ctas=st.integers(1, 3),
       phases=st.lists(st.sampled_from(PHASES), min_size=1, max_size=3), seed=st.integers(0, 10**6),
       base=st.sampled_from([0, 40, 2**32 - 3, 2**32 - 17]))
@settings(max_examples=200, deadline=None)
def test_rsag_protocol_is_race_free_and_deadlock_free(world, n_chunks, ctas, phases, seed, base):
    C = hpc_patterns_b200.native()
    end = simulate(world, n_chunks, ctas, phases, seed, epoch_base=base)
    advance = sum(C.rsag_epoch_advance(_phase_id(C, p), world) for p in phases)
    assert end == (base + advance) & 0xFFFFFFFF


@pytest.mark.parametrize("phase", PHASES)
@pytest.mark.parametrize("world", range(1, 10))
def test_every_phase_at_every_world(world, phase):
    simulate(world, 3, 2, [phase, phase], seed=world, epoch_base=2**32 - world)


@pytest.mark.parametrize("world", range(1, 10))
def test_epoch_advance_and_segment_owner(world):
    C = hpc_patterns_b200.native()
    assert C.rsag_epoch_advance(C.RSAG_ALLREDUCE, world) == 2 * (world - 1)
    assert C.rsag_epoch_advance(C.RSAG_REDUCE_SCATTER, world) == world - 1
    assert C.rsag_epoch_advance(C.RSAG_ALL_GATHER, world) == world - 1
    for r in range(world):
        assert C.rsag_segment(world - 1, r, world) == r              # the hop that finishes a segment is its owner's


def _caught(mutation, worlds, phases_list, seeds=40):
    hits = 0
    for world in worlds:
        for phases in phases_list:
            for seed in range(seeds):
                try:
                    simulate(world, 3, 2, phases, seed, epoch_base=7, mutation=mutation)
                except Violation:
                    hits += 1
                    break
            else:
                return False, (world, phases)
    return hits > 0, None


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_caught(mutation):
    """The model is not vacuous: every broken rule is found at every world size where it changes anything."""
    if mutation == "wait_one_early":
        ok, where = _caught(mutation, range(2, 7), [["allreduce"], ["reduce_scatter"], ["all_gather"]])
    elif mutation == "forward_own_va":           # only hops 1 .. P-2 forward a partial sum
        ok, where = _caught(mutation, range(3, 8), [["allreduce"], ["reduce_scatter"]])
    elif mutation == "push_into_right_own_segment":
        ok, where = _caught(mutation, range(2, 8), [["allreduce"], ["all_gather"]])
    else:
        ok, where = _caught(mutation, range(2, 8), [["allreduce"], ["reduce_scatter"], ["all_gather"]])
    assert ok, f"{mutation} not caught at {where}"


# ------------------------------------------------------------------------------------------------ oracle ----
def _numpy_rsag(vas):
    world, n = len(vas), vas[0].numel()
    a = [v.numpy() for v in vas]
    out = np.empty_like(a[0])
    seg_n = n // world
    for s in range(world):
        lo = s * seg_n
        for i in range(lo, lo + seg_n):
            acc = a[(s + 1) % world][i]
            for k in range(2, world + 1):
                acc = (acc + a[(s + k) % world][i]).astype(a[0].dtype)
            out[i] = acc
    return torch.from_numpy(out)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_rsag_expected_agrees_with_a_numpy_loop(world, dtype):
    n = world * (16 // TORCH_DTYPE[dtype].itemsize) * 3
    vas = make_inputs(world, n, dtype, seed=world)
    with np.errstate(over="ignore"):
        want = _numpy_rsag(vas)
    assert mismatches(rsag_expected(vas), want.view(TORCH_DTYPE[dtype])) == 0
    for s in range(world):
        seg = slice(s * n // world, (s + 1) * n // world)
        assert mismatches(reduce_scatter_expected(vas, s), rsag_expected(vas)[seg]) == 0


@pytest.mark.parametrize("world", [3, 4, 5, 8])
def test_rsag_order_differs_from_the_fused_ring(world):
    """For random floats the pinned order is visible: the result differs from every rank's fused-ring result."""
    vas = make_inputs(world, world * 4 * 256, "float", seed=11)
    got = rsag_expected(vas)
    for r in range(world):
        assert mismatches(got, ring_expected(vas, r)) > 0


# --------------------------------------------------------------------------------- bin/allreduce --cpu ----
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_host_thread_twin(bin_dir, world, dtype, tmp_path):
    rows = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "allreduce"), "--cpu", "--algo", "ring-rsag", "-n", str(world), "-p",
                        "9", "--type", dtype, "--json", str(rows)], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == world and "FAILED" not in p.stdout
    assert "host-ring-rsag" in p.stdout
    import json

    row = json.loads(rows.read_text().splitlines()[-1])
    unit = 16 // TORCH_DTYPE[dtype].itemsize * world
    assert row["algo"] == "host-ring-rsag" and row["mismatches"] == 0
    assert row["elements"] % unit == 0 and 512 <= row["elements"] < 512 + unit


@pytest.mark.parametrize("args", [["--slots", "2"], ["--pull"], ["--cpu", "--slots", "2"], ["--cpu", "--pull"]])
def test_usage_errors(bin_dir, args):
    p = subprocess.run([os.path.join(bin_dir, "allreduce"), "--algo", "ring-rsag", *args], capture_output=True,
                       text=True, timeout=60)
    assert p.returncode == 1 and "not of ring-rsag" in p.stderr, p.stdout + p.stderr


def test_unknown_algo_still_rejected(bin_dir):
    p = subprocess.run([os.path.join(bin_dir, "allreduce"), "--cpu", "--algo", "ring-rsa"], capture_output=True,
                       text=True, timeout=60)
    assert p.returncode == 1 and "unknown --algo ring-rsa" in p.stderr
