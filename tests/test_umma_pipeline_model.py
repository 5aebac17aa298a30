"""Executable model of the mbarrier pipeline of the tensor-core tile loop (csrc/kernels/wgmma.cuh: gemm_persistent),
on the CPU.

A protocol error in the tile loop is a hang or silently wrong data.  This model re-states its barrier protocol — who
initialises which barrier with which count, who arrives / expects bytes / waits on which parity — with mbarrier
semantics (pending arrivals, transaction bytes, phase bit), runs the producer warp and the two consumer warpgroups of
each CTA (one CTA, or a pair sharing the B tile by TMA multicast) as coroutines under a random scheduler in which every
asynchronous completion (TMA bytes landing, wgmma groups retiring) is delayed arbitrarily, and checks: no deadlock,
no MMA on a stage whose bytes have not all landed, no stage refilled (in either CTA of a pair) while a consumer still
holds it.  The consumers release a stage after ``wgmma.wait_group 1`` has retired the k-block that read it, with a
remote ``mbarrier.arrive`` into every CTA of the pair; the empty barriers count 2 x kConsumers arrivals in a pair.
Mutated protocols (a wrong arrival count, a missing remote arrive, a release before the MMA retired, a short
transaction count) must be caught.
"""
import random

import pytest


class ProtocolError(Exception):
    pass


class MBar:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.tx, self.phase = name, count, count, 0, 0

    def _maybe_flip(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self, expect_tx=0):
        if self.pending == 0:
            raise ProtocolError(f"{self.name}: arrival on a phase whose arrivals are already complete")
        self.tx += expect_tx
        self.pending -= 1
        self._maybe_flip()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._maybe_flip()

    def done(self, parity):  # mbarrier.try_wait.parity: has the phase with this parity completed?
        return (self.phase & 1) != parity


def run(agents, pending_events, rng, max_steps=200000):
    """agents: generators that yield a zero-argument predicate to wait on (or None to just yield the CPU).
    pending_events: list of callables (async completions) that the scheduler fires at random times, FIFO per queue."""
    waiting = {a: None for a in agents}
    steps = 0
    while waiting:
        steps += 1
        if steps > max_steps:
            raise ProtocolError("livelock")
        choices = [("agent", a) for a, cond in waiting.items() if cond is None or cond()]
        choices += [("event", q) for q in pending_events if q]
        if not choices:
            raise ProtocolError("deadlock: " + ", ".join(sorted(a.gi_code.co_name + str(a.gi_frame.f_locals.get("cta", ""))
                                                               for a in waiting)))
        kind, x = rng.choice(choices)
        if kind == "event":
            x.pop(0)()
            continue
        try:
            waiting[x] = next(x)
        except StopIteration:
            del waiting[x]
    for q in pending_events:
        while q:
            q.pop(0)()


A_BYTES, B_BYTES = 16384, 32768
CONSUMERS = 2


def simulate_wgmma(num_items, num_kb, stages, seed, cluster=2, empty_count=None, remote_release=True,
                   release_before_retire=False, expect_bytes=A_BYTES + B_BYTES):
    rng = random.Random(seed)
    empty_count = CONSUMERS * cluster if empty_count is None else empty_count
    full = [[MBar(f"full[{c}][{s}]", 1) for s in range(stages)] for c in range(cluster)]
    empty = [[MBar(f"empty[{c}][{s}]", empty_count) for s in range(stages)] for c in range(cluster)]
    landed = {}                                        # (cta, stage, fill) -> bytes landed for that fill
    holders = [[0] * stages for _ in range(cluster)]   # consumers that acquired stage s of cta c and not released it
    reading = [[0] * stages for _ in range(cluster)]   # issued wgmma groups on stage s of cta c not yet retired
    tma_q = [[] for _ in range(cluster)]
    mma_q = [[[] for _ in range(CONSUMERS)] for _ in range(cluster)]   # wgmma groups retire in order, per warpgroup
    outstanding = [[0] * CONSUMERS for _ in range(cluster)]

    def producer(cta):
        stage, phase, t = 0, 0, 0
        for _ in range(num_items):
            for _ in range(num_kb):
                yield lambda s=stage, p=phase: empty[cta][s].done(p ^ 1)
                for d in range(cluster):                   # my half of B lands in every CTA of the pair
                    if holders[d][stage] or reading[d][stage]:
                        raise ProtocolError(f"cta {cta} refills stage {stage} while cta {d} still uses it")
                full[cta][stage].arrive(expect_tx=expect_bytes)
                own_bytes = A_BYTES + (B_BYTES if cluster == 1 else 0)

                def own(s=stage, c=cta, n=t // stages, b=own_bytes):
                    landed[c, s, n] = landed.get((c, s, n), 0) + b
                    full[c][s].complete_tx(b)

                def half_b(s=stage, n=t // stages):
                    for d in range(cluster):
                        landed[d, s, n] = landed.get((d, s, n), 0) + B_BYTES // 2
                        full[d][s].complete_tx(B_BYTES // 2)

                tma_q[cta] += [own] + ([half_b] if cluster > 1 else [])
                t += 1
                stage += 1
                if stage == stages:
                    stage, phase = 0, phase ^ 1

    def release(cta, s):
        holders[cta][s] -= 1
        for d in (range(cluster) if remote_release else [cta]):
            empty[d][s].arrive()

    def consumer(cta, g):
        stage, phase, t = 0, 0, 0
        for _ in range(num_items):
            prev = None
            for _ in range(num_kb):
                yield lambda s=stage, p=phase: full[cta][s].done(p)
                got = landed.get((cta, stage, t // stages), 0)
                if got != A_BYTES + B_BYTES:
                    raise ProtocolError(f"cta {cta}: MMA on stage {stage} with {got} bytes landed")
                holders[cta][stage] += 1
                reading[cta][stage] += 1
                outstanding[cta][g] += 1

                def retired(c=cta, w=g, s=stage):
                    outstanding[c][w] -= 1
                    reading[c][s] -= 1

                mma_q[cta][g].append(retired)
                if release_before_retire:
                    release(cta, stage)
                    prev = None
                else:
                    yield lambda c=cta, w=g: outstanding[c][w] <= 1       # wgmma.wait_group 1
                    if prev is not None:
                        release(cta, prev)
                    prev = stage
                t += 1
                stage += 1
                if stage == stages:
                    stage, phase = 0, phase ^ 1
            yield lambda c=cta, w=g: outstanding[c][w] == 0               # wgmma.wait_group 0
            if prev is not None:
                release(cta, prev)
            yield None                                                     # the epilogue stores the tile

    agents = [producer(c) for c in range(cluster)] + [consumer(c, g) for c in range(cluster) for g in range(CONSUMERS)]
    run(agents, tma_q + [q for per_cta in mma_q for q in per_cta], rng)
    return True


@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("num_items,num_kb", [(1, 1), (1, 7), (2, 3), (3, 6), (5, 13), (4, 1)])
def test_wgmma_pipeline_has_no_deadlock_and_no_hazard(num_items, num_kb, cluster):
    for seed in range(25):
        assert simulate_wgmma(num_items, num_kb, stages=4, seed=seed, cluster=cluster)


@pytest.mark.parametrize("mutation", [dict(empty_count=2), dict(empty_count=3), dict(remote_release=False),
                                      dict(release_before_retire=True), dict(expect_bytes=A_BYTES + B_BYTES // 2)])
def test_checker_catches_broken_protocols(mutation):
    """Not vacuous: each of these one-line protocol errors is reported (as a deadlock or as a hazard)."""
    caught = 0
    for seed in range(40):
        try:
            simulate_wgmma(4, 5, stages=4, seed=seed, **mutation)
        except ProtocolError:
            caught += 1
    assert caught > 0, mutation
