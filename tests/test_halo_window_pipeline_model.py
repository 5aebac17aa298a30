"""Executable model of the role-split pipeline inside one K-halo CTA (csrc/kernels/halo_stencil.cu), on the CPU.

The kernel has three roles.  A producer thread streams the R + 2 tiles of a column in boundary-first order (row R-1, up
halo, row 0, down halo, rows 1 .. R-2) into an input ring guarded by `full` / `empty` mbarriers.  The math warps read
each input tile once into a register window (up, centre, and the saved row R-1 and down halo), free the slot, and
write the results of rows 0 .. R-1 into an output staging ring (`ofull` / `oempty`).  A store thread sends each output
slot to global memory, keeps up to two stores reading shared memory (one when the ring has two slots) and frees a
slot once `bulk_wait_read` has seen its store read; at the end of a step it waits for all its stores to be performed (`bulk_wait<0>`), publishes the step word and arrives on the CTA-local `stored` barrier, which the
producer waits on before it loads the next step (the next step reads what this one wrote).

This model restates exactly those rules — cursors, barrier counts and parities, the window — and runs the producer,
the store thread and the math warps as coroutines under a random scheduler that delays every asynchronous completion
(a load landing, a store reading its slot, a store being performed in global memory) arbitrarily.  Global memory holds
a version per (buffer, row, column); a load reads it when it lands and a store writes it when it is performed.  So
both the in-CTA races and the cross-step RAW / WAR order through global memory are checked.  Checked under every
schedule: no deadlock, no arrival on a completed barrier phase, every stencil sees rows r-1, r, r+1 of its own step
and column, every result is stored exactly once, no load lands in a slot that a math warp still has to read, and no
math warp writes an output slot that a store is still reading.  Mutated rules must be caught.
"""
import random

import pytest

from tests.test_umma_pipeline_model import MBar, ProtocolError, run

MATH_WARPS = 2


class Cursor:
    """`struct Ring` of the kernel: slot index + phase parity of its current use."""

    def __init__(self, stages):
        self.slot, self.phase, self.S = 0, 0, stages

    def advance(self):
        self.slot += 1
        if self.slot == self.S:
            self.slot, self.phase = 0, self.phase ^ 1


def load_row(q, R):
    """halo_load_row() of the kernel: the row of the q-th load of a column (-1 up halo, R down halo)."""
    if q == 0:
        return R - 1
    if q == 1:
        return -1
    if R == 1:
        return 1
    if q == 2:
        return 0
    if q == 3:
        return R
    return q - 3


def simulate(in_stages, out_stages, rows, ncols, steps, seed, self_neighbour=True, empty_count=MATH_WARPS,
             free_out_early=False, swap_saved=False, skip_stored_wait=False):
    """self_neighbour: N = 1 pull, the halos are this CTA's own rows R-1 and 0 and the step word is its own; otherwise
    the halos come from neighbours whose rows are always ready and no word is modelled (the N > 1 case in which the
    words say nothing about this CTA's own stores).  The other keywords are mutations; the defaults are the kernel's."""
    rng = random.Random(seed)
    R, W = rows, MATH_WARPS
    full = [MBar(f"full[{i}]", 1) for i in range(in_stages)]
    empty = [MBar(f"empty[{i}]", empty_count) for i in range(in_stages)]
    ofull = [MBar(f"ofull[{i}]", W) for i in range(out_stages)]
    oempty = [MBar(f"oempty[{i}]", 1) for i in range(out_stages)]
    stored = MBar("stored", 1)
    word = [0]
    mem = {(0, r, c): 0 for r in range(R) for c in range(ncols)}   # (buffer, row, column) -> step whose input it is
    in_tile = [None] * in_stages       # (column, row, version) of the tile in the slot
    unread = [0] * in_stages           # math warps that still have to read the slot's tile
    out_parts = [dict() for _ in range(out_stages)]    # warp -> (step, column, row) it wrote into the slot
    reading = [0] * out_stages         # stores issued on the slot that have not read it yet
    load_q, read_q, perf_q = [], [], []
    done = []

    def producer():
        ld = Cursor(in_stages)
        for g in range(steps):
            if g > 0 and not skip_stored_wait:
                yield lambda p=(g - 1) & 1: stored.done(p)
            if self_neighbour:
                yield lambda g=g: word[0] >= g
            for col in range(ncols):
                for q in range(R + 2):
                    row = load_row(q, R)
                    yield lambda s=ld.slot, p=ld.phase ^ 1: empty[s].done(p)
                    slot = ld.slot
                    full[slot].arrive(expect_tx=1)

                    def landed(slot=slot, g=g, col=col, row=row):
                        if unread[slot]:
                            raise ProtocolError(f"load of step {g} col {col} row {row} landed in slot {slot}: "
                                                f"{in_tile[slot]} is still being read")
                        if row in (-1, R) and not self_neighbour:
                            ver = g
                        else:
                            own = R - 1 if row == -1 else 0 if row == R else row
                            ver = mem.get((g & 1, own, col))
                        in_tile[slot] = (col, row, ver)
                        unread[slot] = W
                        full[slot].complete_tx(1)

                    load_q.append(landed)
                    ld.advance()

    def store_thread():
        st = Cursor(out_stages)
        lag = 2 if out_stages >= 3 else 1
        for g in range(steps):
            outstanding = []
            for col in range(ncols):
                for r in range(R):
                    yield lambda s=st.slot, p=st.phase: ofull[s].done(p)
                    slot = st.slot
                    reading[slot] += 1
                    tok = {"read": False, "performed": False}

                    def read_out(slot=slot, want=(g, col, r), tok=tok):
                        got = [out_parts[slot].get(w) for w in range(W)]
                        if any(x != want for x in got):
                            raise ProtocolError(f"store of {want} read {got} from output slot {slot}")
                        reading[slot] -= 1
                        tok["read"] = True
                        done.append(want)

                        def performed(want=want, tok=tok):
                            g_, col_, r_ = want
                            mem[((g_ + 1) & 1, r_, col_)] = g_ + 1
                            tok["performed"] = True

                        perf_q.append(performed)

                    read_q.append(read_out)
                    outstanding.append(tok)
                    if free_out_early:
                        oempty[slot].arrive()
                    else:
                        # bulk_wait_read<lag>: every store but the `lag` newest has read its slot; free the one before
                        yield lambda older=list(outstanding[:-lag]): all(t["read"] for t in older)
                        if len(outstanding) > lag:
                            oempty[(slot - lag) % out_stages].arrive()
                    st.advance()
            yield lambda ts=list(outstanding): all(t["performed"] for t in ts)     # bulk_wait<0>
            if not free_out_early:
                for k in range(min(lag, len(outstanding)), 0, -1):
                    oempty[(st.slot - k) % out_stages].arrive()
            word[0] = g + 1
            stored.arrive()

    def math(w):
        inp, out = Cursor(in_stages), Cursor(out_stages)

        def take():
            slot = inp.slot
            tile = in_tile[slot]
            unread[slot] -= 1
            return slot, tile

        def release(slot):
            empty[slot].arrive()
            inp.advance()

        def read():
            yield lambda s=inp.slot, p=inp.phase: full[s].done(p)
            slot, tile = take()
            yield None
            release(slot)
            return tile

        def put(g, col, r, up, ce, dn):
            slot = out.slot
            if reading[slot]:
                raise ProtocolError(f"warp {w} wrote output slot {slot} while a store still reads it")
            want = ((col, r - 1, g), (col, r, g), (col, r + 1, g))
            if (up, ce, dn) != want:
                raise ProtocolError(f"stencil of step {g} col {col} row {r} (warp {w}) read {(up, ce, dn)}")
            out_parts[slot][w] = (g, col, r)

        def publish():
            ofull[out.slot].arrive()
            out.advance()

        def write(g, col, r, up, ce, dn):
            yield lambda s=out.slot, p=out.phase ^ 1: oempty[s].done(p)
            put(g, col, r, up, ce, dn)
            yield None
            publish()

        def read_write(g, col, r, up, ce):
            yield lambda s=inp.slot, p=inp.phase: full[s].done(p)
            yield lambda s=out.slot, p=out.phase ^ 1: oempty[s].done(p)
            slot, dn = take()
            put(g, col, r, up, ce, dn)
            yield None
            release(slot)
            publish()
            return dn

        for g in range(steps):
            for col in range(ncols):
                last = yield from read()
                up = yield from read()
                if R == 1:
                    dnh = yield from read()
                    if swap_saved:
                        last, dnh = dnh, last
                    yield from write(g, col, 0, up, last, dnh)
                    continue
                ce = yield from read()
                dnh = yield from read()
                if swap_saved and R == 2:
                    last, dnh = dnh, last
                for r in range(R - 2):
                    dn = yield from read_write(g, col, r, up, ce)
                    up, ce = ce, dn
                yield from write(g, col, R - 2, up, ce, last)
                yield from write(g, col, R - 1, ce, last, dnh)

    agents = [producer(), store_thread()] + [math(w) for w in range(W)]
    run(agents, [load_q, read_q, perf_q], rng)
    want = [(g, c, r) for g in range(steps) for c in range(ncols) for r in range(R)]
    if sorted(done) != sorted(want) or len(done) != len(set(done)):
        raise ProtocolError("not every result was stored exactly once")
    return len(done)


@pytest.mark.parametrize("in_stages,out_stages", [(1, 2), (2, 2), (3, 3), (9, 3)])
@pytest.mark.parametrize("rows,ncols", [(1, 3), (2, 2), (3, 3), (4, 2), (8, 2)])
@pytest.mark.parametrize("self_neighbour", [True, False], ids=["n1", "n_gt_1"])
def test_kernel_rules_are_safe_under_random_schedules(in_stages, out_stages, rows, ncols, self_neighbour):
    for seed in range(20):
        assert simulate(in_stages, out_stages, rows, ncols, steps=3, seed=seed,
                        self_neighbour=self_neighbour) == 3 * rows * ncols


def _caught(seeds=300, match=None, **kw):
    with pytest.raises(ProtocolError, match=match):
        for seed in range(seeds):
            simulate(seed=seed, **kw)


def test_input_slot_freed_before_every_warp_read_it_is_caught():
    """`empty` counting one arrival instead of one per math warp: the first warp's release frees the slot."""
    _caught(in_stages=2, out_stages=2, rows=3, ncols=3, steps=2, empty_count=1)


def test_output_slot_reused_before_its_store_read_it_is_caught():
    """The store thread frees a slot as soon as it issued the store, without bulk_wait_read."""
    _caught(in_stages=4, out_stages=2, rows=3, ncols=3, steps=2, free_out_early=True, match="still reads")


@pytest.mark.parametrize("rows", [1, 2])
def test_saved_halo_used_for_the_wrong_row_is_caught(rows):
    """At R = 1 and 2 the saved row R-1 and the saved down halo are both consumed by the last rows; swapping them."""
    _caught(seeds=5, in_stages=3, out_stages=2, rows=rows, ncols=2, steps=1, swap_saved=True, match="stencil of")


def test_output_ring_one_slot_too_short_deadlocks():
    """The store thread frees its newest slot only after a later store: one output slot can never be refilled."""
    _caught(seeds=1, in_stages=4, out_stages=1, rows=3, ncols=2, steps=1, match="deadlock")


def test_producer_starting_a_step_before_its_own_stores_are_performed_is_caught():
    """Without the CTA-local `stored` barrier the next step can read a row before this CTA's store of it is performed.
    At N > 1 nothing else orders the two (the neighbours' words only speak for the neighbours)."""
    _caught(seeds=400, in_stages=9, out_stages=3, rows=3, ncols=2, steps=3, self_neighbour=False,
            skip_stored_wait=True, match="stencil of")


def test_own_step_word_orders_the_steps_at_n1():
    """At N = 1 the CTA's own step word already orders the steps: the same mutation is harmless there."""
    for seed in range(50):
        assert simulate(9, 3, 3, 2, steps=3, seed=seed, self_neighbour=True, skip_stored_wait=True) == 18
