"""RowParallelLinear, ColumnParallelLinear and ParallelMLP on virtual ranks of one GPU, step after step, against fp64.

Several ranks of one process share the GPU: their symmetric buffers and signal pads come from a ``LocalGroup`` (peer
pointers are plain pointers), each rank enqueues on its own stream (a rank's device barrier must not wait for arrivals
queued behind it), and every rank's grid is capped at SMs / world so that all persistent grids are resident at once.
Every step draws new activations and new weights on every rank (tests/tp_oracle.py), and all steps are enqueued
without a host synchronisation between them (and without a device allocation, an implicit one): a layer that gathers last step's rows, adds into a shard nobody zeroed,
waits for the wrong ready count or publishes the wrong epoch or ticket fails here.

* A. RowParallelLinear at 1, 2, 3, 4, 5, 8 ranks, 1-3 tile rows per shard, N/256 in {1, 3}, K_local/64 in {1, 3, 64},
  cluster 0, 1 and 2 (2 with two tile rows per shard, which CTA pairs need), the co-resident grid and 1 or 3 CTAs:
  REDG and TMA epilogues bit for bit against the fp64 sum over ranks; bf16 shards one of the outcomes of the P
  roundings in some order (within the summation bound above 4 ranks).  After every step, on every rank: status OK,
  the done words PAD_DONE + q hold the epoch, the ticket word is ``ticket_issued`` mod 2^32.
* B. ColumnParallelLinear at 1-8 ranks, chunks of 0 (4096), 512, 2048, 4096 bytes, every activation with fp32 and bf16
  output (none / relu bit for bit, gelu / silu within ``activation_bound``, plus half a bf16 ulp for bf16), y filled
  with NaN before every step; steps alternate ``forward(x)`` and ``wait_readers()`` + a write into ``x_local`` +
  ``forward(None)``.  After every step: the gathered A is this step's rows of every rank, every peer block's ready
  counter equals ``ready_base``, the rank's own blocks are unchanged, the ticket word is ``ticket_issued`` mod 2^32.
* C. ParallelMLP at 1, 2, 4, 8 ranks with relu, gelu and silu, three steps: the hidden values against the epilogue's
  activation of the exact C; the block output against the fp64 product of the kernel's own hidden values summed over
  ranks, bit for bit on the exact case (tests/gemm_oracle.py::mlp_exact_operands), else within ffn 2^-22 sum |h| |w|.
* D. Ticket words and ready counters started a few launches before 2^32, five exact steps across the wrap.
* E. Planted faults: a shard that is not zeroed, rows not copied into ``x_local``: the checks report them.
* F. ``python -m hpc_patterns_b200 tp --check --mlp`` at one rank exits 0 with every verdict true.
"""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
from tests.gemm_oracle import activation_bound, describe, mismatches, rne_bf16, shard_problems
from tests.tp_oracle import (COLUMN_CASES, MAX, MLP_CASES, MLP_STEPS, ROW_CASES, STEPS, ColumnCase, RowCase,
                             column_step, mlp_hidden, mlp_output, mlp_step, row_expected, row_step)

pytestmark = pytest.mark.gpu

DEV = 0
F32, BF16 = torch.float32, torch.bfloat16
TIMEOUT_S = 10.0             # a protocol fault ends as a timeout status, never as a hang
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 0xFFFFFFFF


@pytest.fixture(scope="module")
def native():
    assert torch.cuda.is_available()
    torch.cuda.set_device(DEV)
    C = hpc_patterns_b200.native()
    _first_launches(C)
    return C


def _first_launches(C):
    """Launch every kernel the layers use once, on one rank, with nothing else running on the device.

    The first launch of a kernel in a process can wait for the device to go idle.  Seen on an H100 after other
    processes had used it: rank 0's first launch of the CTA-pair TMA-reduce kernel, enqueued behind its own spinning
    device barrier, waited for rank 1's arrival, which the one host thread had not enqueued yet, until the barrier's
    deadline; rank 0 then added into rank 1's shard before rank 1 zeroed it.  One process per GPU never waits so."""
    from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_reduce_scatter
    from hpc_patterns_b200.parallel.local import LocalGroup

    a = torch.zeros(256, 64, dtype=BF16, device=DEV)
    for cluster in (1, 2):
        for out, epilogue in ((F32, "red"), (F32, "tma"), (BF16, "red")):
            shard = torch.zeros(256, 256, dtype=out, device=DEV)
            gemm_reduce_scatter(a, a, [shard], 0, ctas=2, cluster=cluster, out_dtype=out, epilogue=epilogue)
        for out in (F32, BF16):
            allgather_gemm(a, [a], a, torch.empty(256, 256, dtype=out, device=DEV), 0, ctas=2, cluster=cluster)
    pads = LocalGroup(1, [DEV]).pads()[0]
    pads.device_barrier(torch.cuda.current_stream(DEV).cuda_stream)
    C.wait_flags(pads.word(0, C.PAD_DONE), 1, 0, pads.timeout_ns, pads.status_ptr,
                 torch.cuda.current_stream(DEV).cuda_stream)
    torch.cuda.synchronize(DEV)
    pads.check()
    pads.close()


def _ctas(ctas, world, cluster):
    """The co-resident maximum (even for CTA pairs), or the given number."""
    if ctas != MAX:
        return ctas
    c = max(1, torch.cuda.get_device_properties(DEV).multi_processor_count // world)
    return max(2, c & ~1) if cluster == 2 else c


class _Ranks:
    """``world`` virtual ranks: a LocalGroup, one stream per rank, the group's buffers (closed at the end)."""

    def __init__(self, world):
        from hpc_patterns_b200.parallel.local import LocalGroup

        self.world = world
        self.group = LocalGroup(world, [DEV] * world)
        self.streams = [torch.cuda.Stream(DEV) for _ in range(world)]

    def pads(self):
        return self.group.pads(timeout_s=TIMEOUT_S)

    def symmetric(self, nbytes):
        return self.group.symmetric(nbytes, zero=True)

    def run(self, fn):
        """fn(r) for every rank, each under its own stream."""
        out = []
        for r in range(self.world):
            with torch.cuda.stream(self.streams[r]):
                out.append(fn(r))
        return out

    def synchronize(self):
        for st in self.streams:
            st.synchronize()


def _pad_words(pads):
    """This rank's signal pad as int32 words (done words, ticket, status)."""
    from hpc_patterns_b200.parallel.symmetric import tensor_from_ptr

    return tensor_from_ptr(pads.buf.local_ptr, pads.buf.nbytes, DEV, torch.int32)


def _empty_like(*ts):
    """Where a step's results are saved, allocated before any launch: a device allocation between two ranks'
    launches is an implicit synchronisation, which would hold one rank's kernels behind another rank's spinning ones
    until the deadline."""
    return [torch.empty_like(t) for t in ts]


def _start_tickets(native, layer, start):
    layer.pads.ticket_issued = start
    native.write_u32(layer.pads.ticket_ptr, start & U32)


def _status_and_ticket(native, words, issued, who):
    problems = []
    if int(words[native.PAD_WORDS]) != native.STATUS_OK:
        problems.append(f"{who}: status 0x{int(words[native.PAD_WORDS]) & U32:08x}")
    if int(words[native.PAD_LOCAL]) & U32 != issued & U32:
        problems.append(f"{who}: ticket word {int(words[native.PAD_LOCAL]) & U32} != issued {issued & U32}")
    return problems


# ---- A. RowParallelLinear ------------------------------------------------------------------------------------------
def run_row(native, case: RowCase, steps=STEPS, ticket_start=0, plant=None):
    """``steps`` forwards of ``case`` on virtual ranks; returns one list of problems per step ('' = none)."""
    from hpc_patterns_b200.models.tensor_parallel import RowParallelLinear

    world = case.world
    m, n, k = case.shape
    out = BF16 if case.variant == "bf16" else F32
    ranks = _Ranks(world)
    pads = ranks.pads()
    shards = ranks.symmetric((m // world) * n * (2 if out == BF16 else 4))
    ctas = _ctas(case.ctas, world, case.cluster)
    layers = [RowParallelLinear(ranks.group.comms[r], DEV, m, n, k, cluster=case.cluster, ctas=ctas, out_dtype=out,
                                epilogue="tma" if case.variant == "tma" else "red", timeout_s=TIMEOUT_S,
                                _shared={"pads": pads[r], "shard": shards[r]}) for r in range(world)]
    try:
        for layer in layers:
            if ticket_start:
                _start_tickets(native, layer, ticket_start)
        data = [row_step(case, s, DEV) for s in range(steps)]
        saved = [[_empty_like(layers[r].y, _pad_words(pads[r])) for r in range(world)] for _ in range(steps)]
        torch.cuda.synchronize(DEV)
        got = []
        for s in range(steps):
            xs, ws, _ = data[s]
            if plant is not None and s == 1:                    # a fault from the second step on
                for layer in layers:
                    plant(layer)

            def step(r):
                y, words = saved[s][r]
                layers[r].w.copy_(ws[r])
                y.copy_(layers[r].forward(xs[r]))               # a view of the shard, valid until the next forward
                words.copy_(_pad_words(layers[r].pads))
                return y, words, layers[r].pads.ticket_issued, layers[r].epoch
            got.append(ranks.run(step))
        ranks.synchronize()                                     # status words are judged per step below
        problems = []
        for s in range(steps):
            want = row_expected(data[s][2], world)
            p = []
            for r, (y, words, issued, epoch) in enumerate(got[s]):
                who = f"step {s} rank {r}"
                if out == F32:
                    bad = mismatches(y, want[r].float())
                    if bad:
                        p.append(f"{who}: {bad} elements differ: {describe(y, want[r].float())}")
                else:
                    rows = slice(r * (m // world), (r + 1) * (m // world))
                    shard = shard_problems(y, [c[rows] for c in data[s][2]])
                    if shard:
                        p.append(f"{who}: {shard}")
                done = words[native.PAD_DONE:native.PAD_DONE + world].tolist()
                if done != [epoch] * world:
                    p.append(f"{who}: done words {done}, epoch {epoch}")
                p += _status_and_ticket(native, words, issued, who)
            problems.append("; ".join(p))
        return problems
    finally:
        for layer in layers:
            layer.close()


@pytest.mark.parametrize("case", ROW_CASES, ids=str)
def test_row_parallel_steps_exact(native, case):
    problems = run_row(native, case)
    assert problems == [""] * STEPS, "\n".join(problems)


# ---- B. ColumnParallelLinear ---------------------------------------------------------------------------------------
def run_column(native, case: ColumnCase, out, steps=STEPS, counter_start=0, plant=None):
    """``steps`` forwards alternating the two entry points; one list of problems per step."""
    from hpc_patterns_b200.models.tensor_parallel import ColumnParallelLinear

    world = case.world
    m, n, k = case.shape
    rows = m // world
    ranks = _Ranks(world)
    pads = ranks.pads()
    a_bufs = ranks.symmetric(m * k * 2)
    ctas = _ctas(case.ctas, world, case.cluster)
    layers = [ColumnParallelLinear(ranks.group.comms[r], DEV, m, n, k, out_dtype=out, cluster=case.cluster, ctas=ctas,
                                   chunk_bytes=case.chunk, timeout_s=TIMEOUT_S, activation=case.activation,
                                   _shared={"pads": pads[r], "a": a_bufs[r]}) for r in range(world)]
    try:
        for layer in layers:
            if counter_start:
                _start_tickets(native, layer, counter_start)
                layer.ready_base = counter_start
                layer.ready.fill_(counter_start - (1 << 32) if counter_start >= 1 << 31 else counter_start)
        own0 = [layer.ready.clone() for layer in layers]
        data = [column_step(case, s, DEV) for s in range(steps)]
        saved = [[_empty_like(layer.y, layer.a_full, layer.ready, _pad_words(layer.pads)) for layer in layers]
                 for _ in range(steps + 1)]
        torch.cuda.synchronize(DEV)
        got = []
        for s in range(steps):
            xs, ws, _, _ = data[s]
            if plant is not None and s == 1:                    # a fault from the second step on
                for layer in layers:
                    plant(layer)

            def step(r):
                layer = layers[r]
                y, a_full, ready, words = saved[s][r]
                layer.w.copy_(ws[r])
                layer.y.fill_(float("nan"))                     # a tile nobody wrote shows
                if s % 2 == 0:
                    layer.forward(xs[r])
                else:
                    layer.wait_readers()                        # the peers are done with last step's rows
                    layer.x_local.copy_(xs[r])
                    layer.forward(None)
                for dst, src in ((y, layer.y), (a_full, layer.a_full), (ready, layer.ready),
                                 (words, _pad_words(layer.pads))):
                    dst.copy_(src)
                return y, a_full, ready, layer.ready_base, words, layer.pads.ticket_issued
            got.append(ranks.run(step))

        def last(r):
            layers[r].wait_readers()
            return saved[steps][r][3].copy_(_pad_words(layers[r].pads))
        final = ranks.run(last)
        ranks.synchronize()                                     # status words are judged per step below
        problems = []
        for s in range(steps):
            _, _, a, cs = data[s]
            p = []
            for r, (y, a_full, ready, base, words, issued) in enumerate(got[s]):
                who = f"step {s} rank {r}"
                bad = mismatches(a_full, a)
                if bad:
                    p.append(f"{who}: {bad} elements of the gathered A differ")
                want, bound = activation_bound(cs[r], case.activation)
                if case.activation in ("none", "relu"):
                    want = want.float() if out == F32 else rne_bf16(want)
                    bad = mismatches(y, want)
                    if bad:
                        p.append(f"{who}: {bad} elements differ: {describe(y, want)}")
                else:
                    if out == BF16:                             # + half a bf16 ulp of the fp32 result
                        bound = bound + 2.0 ** -8 * (want.abs() + bound)
                    bad = int((~((y.double() - want).abs() <= bound)).sum())
                    if bad:
                        p.append(f"{who}: {bad} elements outside the bound")
                own = slice(r * rows // 128, (r + 1) * rows // 128)
                peer = torch.ones(m // 128, dtype=torch.bool, device=ready.device)
                peer[own] = False
                counts = ready.long() & U32
                if world > 1 and not bool((counts[peer] == base & U32).all()):
                    p.append(f"{who}: ready counters {counts.tolist()}, ready_base {base & U32}")
                if not torch.equal(ready[own], own0[r][own]):
                    p.append(f"{who}: the rank's own ready counters changed")
                p += _status_and_ticket(native, words, issued, who)
            problems.append("; ".join(p))
        if world > 1:
            for r, words in enumerate(final):
                done = words[native.PAD_DONE:native.PAD_DONE + world].tolist()
                if done != [steps] * world:
                    problems[-1] += f"; after the last step, rank {r}: done words {done}"
        return problems
    finally:
        for layer in layers:
            layer.close()


@pytest.mark.parametrize("case", COLUMN_CASES, ids=str)
def test_column_parallel_steps(native, case):
    for out in (F32, BF16):
        problems = run_column(native, case, out)
        assert problems == [""] * STEPS, f"{out}:\n" + "\n".join(problems)


# ---- C. ParallelMLP ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", MLP_CASES, ids=str)
def test_parallel_mlp_steps(native, case):
    from hpc_patterns_b200.models.tensor_parallel import ParallelMLP

    world = case.world
    tokens, hidden, ffn = case.shape
    ranks = _Ranks(world)
    up_pads, down_pads = ranks.pads(), ranks.pads()
    up_a = ranks.symmetric(tokens * hidden * 2)
    down_shards = ranks.symmetric((tokens // world) * hidden * 4)
    ctas = _ctas(case.ctas, world, 1)
    mlps = [ParallelMLP(ranks.group.comms[r], DEV, tokens, hidden, ffn, activation=case.activation, cluster=1,
                        ctas=ctas, timeout_s=TIMEOUT_S,
                        _shared={"up": {"pads": up_pads[r], "a": up_a[r]},
                                 "down": {"pads": down_pads[r], "shard": down_shards[r]}}) for r in range(world)]
    try:
        data = [mlp_step(case, s, DEV) for s in range(MLP_STEPS)]
        saved = [[_empty_like(mlp.down.y, mlp.up.y) for mlp in mlps] for _ in range(MLP_STEPS)]
        torch.cuda.synchronize(DEV)
        got = []
        for s in range(MLP_STEPS):
            xs, ups, downs, _ = data[s]

            def step(r):
                y, h = saved[s][r]
                mlps[r].up.w.copy_(ups[r])
                mlps[r].down.w.copy_(downs[r])
                y.copy_(mlps[r].forward(xs[r]))
                h.copy_(mlps[r].up.y)
                return y, h
            got.append(ranks.run(step))
        ranks.synchronize()
        for mlp in mlps:
            mlp.check()
        for s in range(MLP_STEPS):
            _, _, downs, cs = data[s]
            hs = [h for _, h in got[s]]
            for r, c in enumerate(cs):
                if case.activation == "relu":
                    want = mlp_hidden(c, "relu")
                    assert mismatches(hs[r], want) == 0, f"step {s} rank {r} hidden: {describe(hs[r], want)}"
                else:
                    want, bound = activation_bound(c, case.activation)
                    bound = bound + 2.0 ** -8 * (want.abs() + bound)
                    bad = int((~((hs[r].double() - want).abs() <= bound)).sum())
                    assert bad == 0, f"step {s} rank {r}: {bad} hidden values outside the bound"
            want, mag = mlp_output(hs, downs, world)         # the kernel's own hidden values: no compounding
            for r, (y, _) in enumerate(got[s]):
                if case.exact:
                    assert mismatches(y, want[r].float()) == 0, f"step {s} rank {r}: {describe(y, want[r].float())}"
                else:
                    bad = int((~((y.double() - want[r]).abs() <= ffn * 2.0 ** -22 * mag[r])).sum())
                    assert bad == 0, f"step {s} rank {r}: {bad} outputs outside ffn 2^-22 sum |h| |w|"
    finally:
        for mlp in mlps:
            mlp.close()


# ---- D. counters across 2^32 ---------------------------------------------------------------------------------------
def test_row_parallel_tickets_wrap(native):
    case = RowCase(4, 1, 1, 3, 1, 5, "red")
    start = (1 << 32) - 2 * 5 - 3                               # the third launch's tickets cross 2^32
    problems = run_row(native, case, steps=5, ticket_start=start)
    assert problems == [""] * 5, "\n".join(problems)


def test_column_parallel_counters_wrap(native):
    case = ColumnCase(4, 512, "none", 5, 1)
    per_launch = native.allgather_gemm_chunks_per_block(case.shape[2], case.chunk)
    start = (1 << 32) - 2 * per_launch - 3                      # ready counters and tickets cross 2^32 on step 3
    assert per_launch > 5
    problems = run_column(native, case, F32, steps=5, counter_start=start)
    assert problems == [""] * 5, "\n".join(problems)


# ---- E. planted faults ---------------------------------------------------------------------------------------------
class _NoMemset:
    """The native module without ``memset_async``: the shard keeps last step's sums."""

    def __init__(self, real):
        self._real = real

    def __getattr__(self, name):
        return (lambda *a, **k: None) if name == "memset_async" else getattr(self._real, name)


def test_row_parallel_reports_a_shard_not_zeroed(native):
    case = RowCase(3, 1, 1, 3, 1, MAX, "red")
    problems = run_row(native, case, plant=lambda layer: setattr(layer, "C", _NoMemset(layer.C)))
    assert problems[0] == ""
    for s in range(1, STEPS):                                   # last step's sums remain in every shard
        for r in range(case.world):
            assert f"step {s} rank {r}: " in problems[s] and " elements differ" in problems[s], problems[s]


def test_column_parallel_reports_rows_not_copied(native, monkeypatch):
    case = ColumnCase(3, 2048, "none", MAX, 1)

    def plant(layer):                                           # the copy lands in a private buffer
        monkeypatch.setattr(layer, "x_local", torch.empty_like(layer.x_local))

    problems = run_column(native, case, F32, plant=plant)
    assert problems[0] == ""
    for s in range(1, STEPS):                                   # every rank gathers last step's rows
        for r in range(case.world):
            assert f"step {s} rank {r}: " in problems[s] and " elements of the gathered A differ" in problems[s]
            assert " elements differ: " in problems[s].split(f"step {s} rank {r}: ", 1)[1], problems[s]


# ---- F. the program at one rank ------------------------------------------------------------------------------------
def test_tp_program_check_at_one_rank():
    env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
    cmd = [sys.executable, "-m", "hpc_patterns_b200", "tp", "--check", "--mlp", "--tokens", "512", "--out-features",
           "512", "--in-features", "256", "--steps", "2"]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    for key in ("row_parallel_exact", "column_parallel_exact", "mlp_within_bound", "mlp_hidden_exact"):
        assert out[key] is True, (key, out)
    assert math.isfinite(out["mlp_max_abs_diff"])
