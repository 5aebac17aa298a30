"""The data movers bit for bit against tests/mover_oracle.py: the copy engines (LdSt, TMA), the fused triad + put
(LdSt, halo LdSt, TMA, the ``halo_ctas`` split, ``l2_hint``), the fused command kernel, the ticket / flag epilogue they
share, the triad payload, and ``FusedTriadExchange`` on one rank.

Every output is a slice of a sentinel-filled buffer with guards on both sides (floats: a NaN with a payload no kernel
produces; bytes: 0xA5), reset to the sentinel before every launch.  Float outputs are compared under the rule of
tests/field_compare.py (bits, NaN as a class), and the sentinel must be found exactly where it is expected, so an
element that was never written is wrong even where a NaN is due.  Guards must keep the sentinel's bits.
"""
import functools

import numpy as np
import pytest
import torch

from tests import mover_oracle as mo
from tests.field_compare import count_wrong

pytestmark = pytest.mark.gpu

G = 64                                    # guard elements (floats: 256 bytes, bytes: 64) on each side
SENT = mo.SENTINEL_BITS
TIMEOUT_NS = int(5e9)


@pytest.fixture(scope="module", autouse=True)
def dev():
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _st():
    return torch.cuda.current_stream().cuda_stream


class Guarded:
    """``n`` elements (float32 or uint8) at ``offset`` elements past a guard of G, inside a sentinel-filled buffer."""

    def __init__(self, n, dtype=torch.float32, offset=0):
        self.n, self.dtype, self.lo = n, dtype, G + offset
        self.buf = torch.empty(self.lo + n + G, dtype=dtype, device="cuda")
        self.reset()

    def reset(self):
        if self.dtype == torch.float32:
            self.buf.view(torch.int32).fill_(SENT)
        else:
            self.buf.fill_(mo.BYTE_SENTINEL)

    @property
    def ptr(self):
        return self.buf.data_ptr() + self.lo * self.buf.element_size()

    def out(self):
        return self.buf[self.lo:self.lo + self.n]

    def guards_intact(self):
        g = torch.cat([self.buf[:self.lo], self.buf[self.lo + self.n:]])
        if self.dtype == torch.float32:
            return bool((g.view(torch.int32) == SENT).all())
        return bool((g == mo.BYTE_SENTINEL).all())


def _dev(x, offset=0):
    """A device copy of a float32 numpy array at ``offset`` floats into a fresh allocation."""
    t = torch.empty(x.size + offset + 8, dtype=torch.float32, device="cuda")
    v = t[offset:offset + x.size]
    v.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    return v


def _check_floats(g, want, what):
    got = g.out().cpu()
    want_t = torch.from_numpy(np.ascontiguousarray(want))
    assert g.guards_intact(), f"{what}: guard overwritten"
    bad = count_wrong(got, want_t)
    # NaN as a class would accept the NaN sentinel where a NaN is due: where the sentinel is, must be exactly where
    # it is expected
    unwritten = int(((got.view(torch.int32) == SENT) != (want_t.view(torch.int32) == SENT)).sum())
    if bad or unwritten:
        idx = np.flatnonzero((got.view(torch.int32) != want_t.view(torch.int32)).numpy())[:4]
        pytest.fail(f"{what}: {bad} wrong, {unwritten} with the sentinel misplaced, of {want.size}; "
                    f"first at {idx.tolist()}: {[hex(int(got.view(torch.int32)[i]) & 0xFFFFFFFF) for i in idx]} want "
                    f"{[hex(int(want_t.view(torch.int32)[i]) & 0xFFFFFFFF) for i in idx]}")


def _sentinel(n):
    return mo.from_bits(np.full(n, SENT, dtype=np.uint32))


@functools.lru_cache(maxsize=64)
def _data(kind, n, s):
    b, c = mo.triad_data(kind, n, s)
    return b, c, mo.fma_f32(b, c, s)


# Three launches per case: every data set once, with a different s each, with and without a put.
LAUNCHES = (("full", 3.0, True), ("cancel", mo.S_VALUES[1], False), ("special", mo.S_VALUES[2], True))
LAUNCHES_SMALL_S = (("full", mo.S_VALUES[3], False), ("cancel", -2.375, True), ("special", mo.S_VALUES[3], True))


def _run_triad(native, engine, tune, n, launches=LAUNCHES, offset=0, what=""):
    local = Guarded(n, offset=offset)
    peer = Guarded(n, offset=offset)
    for kind, s, put in launches:
        b, c, a = _data(kind, n, s)
        db, dc = _dev(b, offset), _dev(c, offset)
        local.reset()
        peer.reset()
        ctas = native.triad_put(local.ptr, peer.ptr if put else 0, db.data_ptr(), dc.data_ptr(), s, n, engine, tune,
                                {}, 0, 0, 0, _st())
        torch.cuda.synchronize()
        assert ctas >= 1
        tag = f"{what} {engine} {tune} n={n} {kind} s={s} put={put}"
        _check_floats(local, a, tag + " local")
        _check_floats(peer, a if put else _sentinel(n), tag + " peer")


TMA_TILE = {None: 4096, 4: 1024, 8: 2048, 16: 4096, 32: 8192}      # stage_kb -> floats per tile


def _sizes(tile):
    return [4, 8, 12, tile - 4, tile, tile + 4, 5 * tile + 4, 37 * tile + 4, (1 << 22) + 8]


LDST_TUNES = [{}, {"unroll": 1}, {"unroll": 2}, {"unroll": 4}, {"vec_bytes": 32}, {"blocked": 1, "ctas": 1},
              {"blocked": 1, "ctas": 3}, {"blocked": 1, "ctas": 37}, {"threads": 32}, {"threads": 96},
              {"threads": 512}, {"vec_bytes": 32, "unroll": 1, "ctas": 3}]
TMA_TUNES = [{}, {"stages": 2}, {"stages": 3}, {"stages": 6}, {"stage_kb": 4}, {"stage_kb": 8}, {"stage_kb": 16},
             {"stage_kb": 32, "stages": 3}, {"stage_kb": 32, "stages": 2}, {"ctas": 1}, {"ctas": 3},
             {"l2_hint": 1}, {"l2_hint": 1, "ctas": 3, "stages": 2}]


TRIAD_CASES = [("ldst", t, n) for t in LDST_TUNES for n in _sizes(4096)] + \
              [("tma", t, n) for t in TMA_TUNES for n in _sizes(TMA_TILE[t.get("stage_kb")])]


@pytest.mark.parametrize("engine,tune,n", TRIAD_CASES, ids=str)
def test_triad_put(native, engine, tune, n):
    """Every tuning at n = 4, 8, 12, one tile - 4, one tile, one tile + 4, 5 and 37 tiles + 4 (far more tiles than
    the 1 or 3 CTAs some tunings pin), 2^22 + 8; a tile is the TMA stage (16 KiB by default)."""
    _run_triad(native, engine, tune, n, launches=LAUNCHES if n % 8 else LAUNCHES_SMALL_S)


def test_triad_put_ldst_wide_fallback_on_16_byte_alignment(native):
    """vec_bytes 32 with pointers that are 16- but not 32-byte aligned takes the 16-byte kernel."""
    for n in (8, 4096 + 8, 5 * 4096 + 8, (1 << 20) + 8):
        _run_triad(native, "ldst", {"vec_bytes": 32}, n, offset=4, what="16-byte aligned")
        _run_triad(native, "ldst", {"vec_bytes": 32, "blocked": 1, "ctas": 3}, n, offset=4, what="16-byte aligned")


def test_triad_put_engines_agree_bit_for_bit(native):
    n = (1 << 22) + 8
    outs = []
    for engine, tune in (("ldst", {}), ("ldst", {"vec_bytes": 32}), ("tma", {}), ("tma", {"stage_kb": 4})):
        for kind, s in (("special", 3.0), ("cancel", mo.S_VALUES[1])):
            b, c, _ = _data(kind, n, s)
            a, db, dc = Guarded(n), _dev(b), _dev(c)
            native.triad_put(a.ptr, 0, db.data_ptr(), dc.data_ptr(), s, n, engine, tune, {}, 0, 0, 0, _st())
            torch.cuda.synchronize()
            outs.append((engine, tune, kind, a.out().view(torch.int32).cpu()))
    for e, t, k, o in outs[2:]:
        ref = outs[0 if k == "special" else 1][3]
        assert torch.equal(o, ref), (e, t, k)


# --------------------------------------------------------------------------------------------------- halo mode ----
HALO_CASES = [("ldst", {}, r) for r in (2, 3, 4)] + [("ldst", {"ctas": 3}, 3)] + \
             [("tma", {}, r) for r in (2, 3, 4)] + \
             [("tma", {"halo_ctas": 4}, r) for r in (2, 3, 4)] + [("tma", {"halo_ctas": 2, "ctas": 6}, 3),
                                                                 ("tma", {"halo_ctas": 1, "ctas": 3}, 4),
                                                                 ("tma", {"l2_hint": 1, "halo_ctas": 3}, 3),
                                                                 ("tma", {"stage_kb": 8, "stages": 4}, 2)]


@pytest.mark.parametrize("engine,tune,ratio", HALO_CASES, ids=str)
def test_triad_put_halo_mode(native, engine, tune, ratio):
    """Only a[:n_put] reaches the peer.  The peer buffer is n long (not n_put), so even a kernel that puts interior
    tiles stays in bounds and is caught by the sentinel after n_put."""
    tile = 4096                                   # 16 KiB: the LdSt halo tile and the default TMA stage
    for n_put in (8 * tile, 3 * tile):
        n = ratio * n_put
        local, peer = Guarded(n), Guarded(n)
        for kind, s, put in LAUNCHES:
            b, c, a = _data(kind, n, s)
            db, dc = _dev(b), _dev(c)          # held until the launch is done
            local.reset()
            peer.reset()
            native.triad_put(local.ptr, peer.ptr if put else 0, db.data_ptr(), dc.data_ptr(), s, n, engine, tune, {},
                             0, 0, 0, _st(), n_put)
            torch.cuda.synchronize()
            tag = f"halo {engine} {tune} ratio={ratio} n_put={n_put} {kind} put={put}"
            _check_floats(local, a, tag + " local")
            _check_floats(peer, mo.triad_expected(b, c, s, n_put=n_put, put=put)[1], tag + " peer")


def test_halo_split_engages(native):
    """The split needs halo_ctas < gridDim.x: the grids used above (and their default) are that large."""
    n_put = 8 * 4096
    for ratio in (2, 3, 4):
        a = Guarded(ratio * n_put)
        b = torch.zeros(ratio * n_put, device="cuda")
        ctas = native.triad_put(a.ptr, 0, b.data_ptr(), b.data_ptr(), 3.0, ratio * n_put, "tma", {"halo_ctas": 4},
                                {}, 0, 0, 0, _st(), n_put)
        torch.cuda.synchronize()
        assert ctas == 8 * ratio > 4


# -------------------------------------------------------------------------------------------------------- copy ----
def _random_bytes(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 255, (n,), dtype=torch.uint8, generator=g)
    return torch.where(x == mo.BYTE_SENTINEL, torch.full_like(x, 0xFF), x)      # no source byte looks unwritten


def _run_copy(native, nbytes, engine, tune, src_is_peer=False, dst_off=0, src_off=0, seed=0):
    src = Guarded(nbytes, torch.uint8, src_off)
    src.out().copy_(_random_bytes(nbytes, seed + nbytes))
    dst = Guarded(nbytes, torch.uint8, dst_off)
    ctas = native.copy(dst.ptr, src.ptr, nbytes, src_is_peer, engine, tune, {}, 0, _st())
    torch.cuda.synchronize()
    tag = f"copy {engine} {tune} {nbytes} B peer={src_is_peer} offsets {dst_off}/{src_off}"
    assert ctas >= 1, tag
    assert dst.guards_intact(), tag + ": guard overwritten"
    got, want = dst.out().cpu(), src.out().cpu()
    if not torch.equal(got, want):
        idx = torch.nonzero(got != want).flatten()
        pytest.fail(f"{tag}: {idx.numel()} wrong bytes, first at {idx[:4].tolist()}")


@pytest.mark.parametrize("engine", ["ldst", "tma"])
def test_copy_every_size_to_80_bytes(native, engine):
    for nbytes in range(0, 81):
        _run_copy(native, nbytes, engine, {})
        if engine == "ldst":
            _run_copy(native, nbytes, engine, {"vec_bytes": 32}, src_is_peer=nbytes % 2 == 1)


@pytest.mark.parametrize("stage_kb", [4, 16])
@pytest.mark.parametrize("engine", ["ldst", "tma"])
def test_copy_around_stage_boundaries(native, engine, stage_kb):
    stage = stage_kb * 1024
    tunes = [{"stage_kb": stage_kb}, {"stage_kb": stage_kb, "ctas": 1}] if engine == "tma" else \
            [{}, {"vec_bytes": 32, "ctas": 3}, {"blocked": 1, "ctas": 5}]
    for tune in tunes:
        for k in (1, 3, 133):
            for d in (-17, -16, -15, -1, 1, 15, 16, 17):
                _run_copy(native, k * stage + d, engine, tune, src_is_peer=d > 0)


def test_copy_ldst_offsets_with_wide_vectors(native):
    """dst / src 0, 16 or 48 bytes past a 256-byte boundary: 32-byte vectors only where both allow it."""
    for dst_off in (0, 16, 48):
        for src_off in (0, 16, 48):
            for nbytes in (31, 4096 + 17, (1 << 20) + 47):
                for peer in (False, True):
                    _run_copy(native, nbytes, "ldst", {"vec_bytes": 32}, peer, dst_off, src_off)


@pytest.mark.parametrize("blocked", [0, 1])
@pytest.mark.parametrize("vec", [16, 32])
@pytest.mark.parametrize("unroll", [1, 2, 4, 8])
def test_copy_ldst_unroll_vector_blocked(native, unroll, vec, blocked):
    for nbytes in (80, 512 * 32 * unroll + 31, (3 << 20) + 29):
        for ctas in (0, 7):
            tune = {"unroll": unroll, "vec_bytes": vec, "blocked": blocked}
            if ctas:
                tune["ctas"] = ctas
            _run_copy(native, nbytes, "ldst", tune, src_is_peer=blocked == 1)


def test_copy_ldst_32_threads_take_a_31_byte_tail(native):
    for nbytes in (31, 63, 32 * 1000 + 31, (1 << 20) + 31):
        _run_copy(native, nbytes, "ldst", {"threads": 32, "vec_bytes": 32})
        _run_copy(native, nbytes, "ldst", {"threads": 32, "vec_bytes": 32, "blocked": 1, "ctas": 3})


@pytest.mark.parametrize("stages", range(2, 9))
def test_copy_tma_stages(native, stages):
    for nbytes in (15, 16 * 1024 * stages + 15, 16 * 1024 * (3 * stages + 1) - 1, (5 << 20) + 13):
        _run_copy(native, nbytes, "tma", {"stages": stages})
        _run_copy(native, nbytes, "tma", {"stages": stages, "ctas": 1}, src_is_peer=True)


# -------------------------------------------------------------------------------------------------------- sync ----
def test_ticket_flag_and_status_over_mixed_launches(native):
    """Copies and triads with mixed engines and CTA counts on one ticket counter: the ticket ends at the sum of the
    returned CTA counts, the flag at the last epoch, the status OK — and every output right."""
    pad = torch.zeros(256, dtype=torch.int32, device="cuda")
    flag = pad.data_ptr() + 4 * native.PAD_DONE
    ticket = pad.data_ptr() + 4 * native.PAD_LOCAL
    status = pad.data_ptr() + 4 * 200
    n = 5 * 4096 + 4
    b, c, a = _data("full", n, 3.0)
    db, dc = _dev(b), _dev(c)
    issued, epoch = 0, 0
    plan = [("copy", "ldst", {}), ("triad", "tma", {"ctas": 3}), ("copy", "tma", {"ctas": 1}),
            ("triad", "ldst", {"blocked": 1, "ctas": 37}), ("copy", "ldst", {"ctas": 5, "vec_bytes": 32}),
            ("triad", "tma", {}), ("triad", "ldst", {})]
    for what, engine, tune in plan:
        epoch += 1
        sync = {"signal_flag": flag, "signal_epoch": epoch, "ticket": ticket, "ticket_base": issued,
                "timeout_ns": TIMEOUT_NS, "status": status}
        if what == "copy":
            src = torch.from_numpy(np.ascontiguousarray(b.view(np.uint8))).cuda()
            dst = Guarded(src.numel(), torch.uint8)
            issued += native.copy(dst.ptr, src.data_ptr(), src.numel(), False, engine, tune, sync, 0, _st())
            torch.cuda.synchronize()
            assert torch.equal(dst.out(), src) and dst.guards_intact()
        else:
            out = Guarded(n)
            issued += native.triad_put(out.ptr, 0, db.data_ptr(), dc.data_ptr(), 3.0, n, engine, tune, sync, 0, 0, 0,
                                       _st())
            torch.cuda.synchronize()
            _check_floats(out, a, f"sync triad {engine} {tune}")
        assert int(pad[native.PAD_LOCAL]) == issued
        assert int(pad[native.PAD_DONE]) == epoch
        assert int(pad[200]) & 0xFFFFFFFF == native.STATUS_OK


# ------------------------------------------------------------------------------------------------- fused bench ----
def _fused_group(native, engine, specs, ctas_mode):
    """specs: ("busy", n, tripcount) | ("triad", n, kind, s) | ("copy", n_floats)."""
    cmds, checks = [], []
    keep = []
    for k, spec in enumerate(specs):
        if spec[0] == "busy":
            _, n, trip = spec
            out = Guarded(n)
            cmds.append({"kind": "busy", "n": n, "tripcount": trip, "a": out.ptr})
            checks.append((out, mo.busy_expected(n, trip), f"busy n={n} trip={trip}"))
        elif spec[0] == "triad":
            _, n, kind, s = spec
            b, c, a = _data(kind, n, s)
            db, dc = _dev(b), _dev(c)
            keep += [db, dc]
            out = Guarded(n)
            cmds.append({"kind": "triad", "n": n, "a": out.ptr, "b": db.data_ptr(), "c": dc.data_ptr(), "s": s})
            checks.append((out, a, f"triad n={n} {kind} s={s}"))
        else:
            _, n = spec
            src = torch.from_numpy(np.ascontiguousarray(mo.triad_data("full", max(n, 1), 3.0, seed=k)[0][:n]))
            dsrc = Guarded(n)
            dsrc.out().copy_(src)
            keep.append(dsrc)
            out = Guarded(n)
            cmds.append({"kind": "copy", "n": n, "dst": out.ptr, "src": dsrc.ptr})
            checks.append((out, src.numpy(), f"copy n={n} ({4 * n % 16} tail bytes)"))
        if ctas_mode == 1:
            cmds[-1]["ctas"] = 1
    total = native.fused_bench(cmds, engine, {}, 0, _st())
    torch.cuda.synchronize()
    assert total >= len(cmds)
    for out, want, tag in checks:
        _check_floats(out, want, f"fused {engine} ctas={ctas_mode} {tag}")


N_BIG = (1 << 20) + 4096
FUSED_GROUPS = {
    "triad-tails": [("triad", N_BIG + r, "special", 3.0) for r in range(4)] + [("triad", r, "full", -2.375)
                                                                               for r in (1, 2, 3)],
    "copy-tails": [("copy", N_BIG + r) for r in range(4)] + [("copy", r) for r in (1, 2, 3)],
    "busy": [("busy", 3000, 0)],
    "busy-triad": [("busy", 700, 2), ("triad", 4099, "cancel", mo.S_VALUES[1])],
    "busy-copy-triad": [("busy", 513, 0), ("copy", 50001), ("triad", 50003, "full", 3.0)],
    "eight": [("busy", 64, 2), ("triad", 5, "special", 3.0), ("copy", 9), ("triad", N_BIG + 2, "cancel", -2.375),
              ("copy", N_BIG + 1), ("busy", 1500, 0), ("triad", 12, "full", mo.S_VALUES[1]), ("copy", 4 * 4096 + 3)],
}


@pytest.mark.parametrize("ctas_mode", [0, 1])
@pytest.mark.parametrize("engine", ["tma", "ldst"])
@pytest.mark.parametrize("group", sorted(FUSED_GROUPS))
def test_fused_bench_groups(native, group, engine, ctas_mode):
    specs = FUSED_GROUPS[group]
    for i in range(0, len(specs), 8):
        _fused_group(native, engine, specs[i:i + 8], ctas_mode)


def test_fused_bench_commands(native):
    """One busy, one copy and one triad command in one group, as the concurrency bench's `fused` mode runs them, on
    both engines: n = 2^21 + 7 runs the triad's n % 4 tail and the copy's 12-byte tail."""
    n = (2 << 20) + 7
    for engine in ("tma", "ldst"):
        _fused_group(native, engine, [("busy", 64, 50), ("copy", n), ("triad", n, "special", 3.0)], 0)


def test_fused_bench_pinned_host_copy_with_tail(native):
    n = (1 << 18) + 3                                              # 12 tail bytes
    h = torch.from_numpy(mo.triad_data("full", n, 3.0)[0]).pin_memory()
    d = Guarded(n)
    back_buf = torch.empty(n + 2 * G, dtype=torch.float32).pin_memory()
    back_buf.view(torch.int32).fill_(SENT)
    for engine in ("tma", "ldst"):
        d.reset()
        back_buf.view(torch.int32).fill_(SENT)
        native.fused_bench([{"kind": "copy", "n": n, "dst": d.ptr, "src": h.data_ptr()}], engine, {}, 0, _st())
        native.fused_bench([{"kind": "copy", "n": n, "dst": back_buf.data_ptr() + 4 * G, "src": d.ptr}], engine, {},
                           0, _st())
        torch.cuda.synchronize()
        _check_floats(d, h.numpy(), f"pinned->device {engine}")
        assert torch.equal(back_buf[G:G + n].view(torch.int32), h.view(torch.int32)), engine
        assert bool((back_buf[:G].view(torch.int32) == SENT).all() and (back_buf[G + n:].view(torch.int32) == SENT)
                    .all()), engine


# ----------------------------------------------------------------------------------------------- the payload ----
def test_fill_triad_inputs_equals_the_reference(native):
    from hpc_patterns_b200.ops.fused import triad_inputs_reference

    n = 3 * 270336 + 1001
    for rank in (0, 1, 5):
        b, c = Guarded(n), Guarded(n)
        native.fill_triad_inputs(b.ptr, c.ptr, n, rank, _st())
        torch.cuda.synchronize()
        rb, rc = triad_inputs_reference(n, rank)
        _check_floats(b, rb.numpy(), f"b rank {rank}")
        _check_floats(c, rc.numpy(), f"c rank {rank}")
        ob, oc = mo.payload(n, rank)
        assert np.array_equal(ob, rb.numpy()) and np.array_equal(oc, rc.numpy())


# ----------------------------------------------------------------------------------------- FusedTriadExchange ----
@pytest.mark.parametrize("ratio", [1, 3])
@pytest.mark.parametrize("engine", ["ldst", "tma"])
def test_fused_exchange_loopback_bit_for_bit(native, engine, ratio):
    """step() and step_from_host with 1, 3 and 8 chunks; the received halo and the local a against the oracle.
    n is not a multiple of 4 * chunks for 3 chunks (both ratios) and 8 chunks (ratio 1)."""
    from hpc_patterns_b200.models.peer2pear import FusedTriadExchange
    from hpc_patterns_b200.parallel.comm import Comm

    nbytes = 16 * 1024 * 13 if ratio > 1 else 16 * 13331
    ex = FusedTriadExchange(Comm(), 0, nbytes=nbytes, engine=engine, compute_ratio=ratio, timeout_s=5.0)
    try:
        n = ex.n
        b, c = mo.payload(ex.n_total, 0)
        want = mo.fma_f32(b, c, 3.0)
        recv = ex.recv.tensor(torch.float32)

        def check(tag):
            got = recv.cpu()
            assert count_wrong(got, torch.from_numpy(want[:n])) == 0, tag
            assert count_wrong(ex.a.cpu(), torch.from_numpy(want)) == 0, tag
            assert ex.verify() == 0, tag

        for _ in range(2):
            recv.view(torch.int32).fill_(SENT)
            ex.a.view(torch.int32).fill_(SENT)
            ex.step()
            torch.cuda.synchronize()
            ex.check()
            check("step")
        host = ex.make_host_input()
        for chunks in (1, 3, 8):
            recv.view(torch.int32).fill_(SENT)
            ex.a.view(torch.int32).fill_(SENT)
            torch.cuda.synchronize()
            assert ex.step_from_host(host, chunks=chunks) == 0
            ex.check()
            check(f"step_from_host chunks={chunks}")
    finally:
        ex.close()


# ------------------------------------------------------------------------------------------- concurrency CLI ----
@pytest.mark.parametrize("commands", [["A"], ["A", "C"]])
def test_concurency_triad_smaller_than_a_vector(native, commands):
    """`A` with 1-3 elements covers no whole vector and launches nothing instead of an empty grid.  The run must
    complete with its report; the exit code is the timing verdict (1 when a 1 µs group is "far from theoretical")."""
    c_params = ["--globalsize_C", "1", "--tripcount_C", "10"] if "C" in commands else []
    for size in ("1", "3"):
        rc, out, err = native.concurency_main(["serial", "--repetitions", "2", "--globalsize_A", size, *c_params,
                                               "--commands", *commands], "cuda")
        assert rc in (0, 1), out + err
        assert out.count("## serial | " + " ".join(commands) + " |") == 1, out + err
        assert "Speedup Relative to Serial" in out and "ERROR" not in out + err, out + err
