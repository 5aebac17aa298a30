"""The stand-alone reduce-scatter (launch_reduce_scatter) on one H100 with virtual ranks, bit for bit against the
owner-first fold of tests/reduce_scatter_oracle.py: every element type with every op it takes, at 1, 2, 3, 4, 5 and 8
ranks, with segments of one 16-byte vector and of a size that runs the main blocks and the tail loop; float and double
sums at segments of 64 MiB.  Each case runs three consecutive launches with fresh data of the oracles' adversarial
kinds and a poisoned receive buffer; the send buffers stay unchanged, the tickets carry across launches and every
status word stays OK.  Then the refusals, and the tensor-level call that enqueues without a host sync."""
import json
import os
import re
import subprocess

import pytest
import torch

import hpc_patterns_b200  # noqa: F401  (at collection, before CUDA starts: asks for eager module loading)
import tests.bitop_oracle as bit
import tests.loc_oracle as loc
import tests.reduce_op_oracle as rop
from hpc_patterns_b200.models.allreduce import ReduceScatterMiniapp, VirtualReduceScatter
from hpc_patterns_b200.ops.allreduce import reduce_scatter, reduce_scatter_reference
from tests.reduce_scatter_oracle import bits_equal, expected, make_inputs

pytestmark = pytest.mark.gpu

_C = hpc_patterns_b200.native()
RS_COUNT_ERROR, RS_WORLD_ERROR = _C.REDUCE_SCATTER_COUNT_ERROR, _C.REDUCE_SCATTER_WORLD_ERROR

LAUNCHES = 3
WORLDS = [1, 2, 3, 4, 5, 8]
CASES = ([(t, op) for t in rop.TYPES for op in ("sum",) + rop.OPS]
         + [(t, op) for t in bit.INT_TYPES for op in bit.BIT_OPS]
         + [(t, op) for t in loc.PAIR_TYPES for op in loc.LOC_OPS])
TAIL_VEC = 2048 + 37        # one whole main block (512 threads x U = 4 vectors) at up to 4 ranks, two at 8, and a tail


def _send(dtype, s):
    """A rank's input as the tensor VirtualReduceScatter.load takes."""
    return torch.frombuffer(bytearray(s), dtype=torch.uint8) if dtype in loc.PAIR_TYPES else s


def _got(dtype, t):
    return bytes(t.numpy().tobytes()) if dtype in loc.PAIR_TYPES else t


def run(world, dtype, op, seg_vec, launches=LAUNCHES, seed=0):
    n = seg_vec * 16 // _C.elem_size(dtype)
    v = VirtualReduceScatter(world, n, dtype, op)
    try:
        for launch in range(launches):
            sends = make_inputs(world, n, dtype, op, seed=1000 * world + seg_vec % 991 + seed, launch=launch)
            v.load([_send(dtype, s) for s in sends])
            for app in v.ranks:     # poison: a result that is never stored cannot pass as the last launch's
                app.recv.tensor().fill_(0xA5 ^ launch)
            torch.cuda.synchronize()
            v.run_once()
            got = v.results()
            for r, app in enumerate(v.ranks):
                want = expected(sends, r, op, dtype)
                bad = bits_equal(_got(dtype, got[r]), want, dtype)
                assert bad == 0, (launch, r, bad)
                sent = app.send.tensor().cpu()
                assert torch.equal(sent, _send(dtype, sends[r]).contiguous().view(torch.uint8).reshape(-1)), \
                    ("send written", launch, r)
            assert [app.pads.ticket_issued for app in v.ranks] == [(launch + 1) * v.ranks[0].launch_ctas] * world
    finally:
        v.close()


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype,op", CASES, ids=[f"{t}-{o}" for t, o in CASES])
def test_every_type_and_op_one_vector(dtype, op, world):
    run(world, dtype, op, 1)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype,op", CASES, ids=[f"{t}-{o}" for t, o in CASES])
def test_every_type_and_op_with_tail(dtype, op, world):
    run(world, dtype, op, TAIL_VEC)


@pytest.mark.parametrize("dtype,op,world", [("float", "sum", 2), ("float", "sum", 4), ("double", "sum", 3)])
def test_large_segments(dtype, op, world):
    run(world, dtype, op, (64 << 20) // 16 + 3, launches=2)


def test_reference_matches_the_oracle_for_the_sum():
    sends = make_inputs(4, 64, "float", "sum", seed=7, launch=0)
    ref = reduce_scatter_reference(sends, "sum", "float")
    assert all(torch.equal(ref[r], expected(sends, r, "sum", "float")) for r in range(4))


def test_refusals(native):
    with pytest.raises(ValueError, match=re.escape(RS_COUNT_ERROR)):
        VirtualReduceScatter(2, 3, "float")
    with pytest.raises(ValueError, match="world <= 8"):
        VirtualReduceScatter(9, 4, "float")
    with pytest.raises(ValueError, match="band reduces integer types only"):
        VirtualReduceScatter(2, 4, "float", "band")
    with pytest.raises(ValueError, match="maxloc reduces value-index pair types only"):
        VirtualReduceScatter(2, 4, "int", "maxloc")
    with pytest.raises(ValueError, match="sum reduces arithmetic types only"):
        VirtualReduceScatter(2, 4, "2int", "sum")
    assert native.reduce_scatter_refusal(17, 4, "float", "sum") == RS_WORLD_ERROR
    assert native.reduce_scatter_refusal(4, 0, "float", "sum") == RS_COUNT_ERROR
    assert native.reduce_scatter_refusal(4, 4, "float", "bxor").endswith("bxor reduces integer types only")
    assert native.reduce_scatter_refusal(4, 4, "int", "bxor") == ""
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    with pytest.raises(ValueError, match="in-place"):     # recv inside my own send buffer (MPI_IN_PLACE)
        reduce_scatter([p, p + 1024], p + 16, [p, p], 0, 0, 0, 4, 1)
    with pytest.raises(ValueError, match="rank out of range"):
        reduce_scatter([p, p + 1024], p + 2048, [p, p], 0, 0, 2, 4, 1)
    with pytest.raises(ValueError, match=RS_WORLD_ERROR):
        reduce_scatter([p] * 17, p, [p] * 17, 0, 0, 0, 4, 1)
    with pytest.raises(ValueError, match="reduces integer types only"):   # the launcher's words, before any launch
        native.reduce_scatter([p, p + 1024], p + 2048, [p, p], 0, 0, 0, 8, 1, dtype="half", op="lor")
    with pytest.raises(Exception, match="in-place"):
        native.reduce_scatter([p, p + 1024], p + 16, [p, p], 0, 0, 0, 4, 1)


def test_tensor_level_call_enqueues_without_host_sync():
    world, n = 4, 4096
    v = VirtualReduceScatter(world, n, "float", "sum")
    try:
        xs = [torch.randn(world * n, device="cuda") for _ in range(world)]
        torch.cuda.synchronize()
        for launch in range(2):
            outs = []
            torch.cuda.set_sync_debug_mode("error")   # any host synchronisation inside the calls raises
            try:
                for app, st, x in zip(v.ranks, v.streams, xs):
                    with torch.cuda.stream(st):
                        outs.append(app.reduce_scatter(x))
            finally:
                torch.cuda.set_sync_debug_mode(0)
            v.synchronize()
            for r in range(world):
                assert torch.equal(outs[r].cpu(), expected([x.cpu() for x in xs], r, "sum", "float")), (launch, r)
    finally:
        v.close()


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("dtype,op", [("float", "sum"), ("bfloat16", "sum"), ("half", "prod"), ("int", "bxor"),
                                      ("ushort", "min"), ("double_int", "minloc")])
def test_cli_four_ranks(bin_dir, tmp_path, dtype, op):
    rows = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "reduce_scatter"), "-n", "4", "-p", "22", "--iters", "3", "--type", dtype,
                        "--op", op, "--json", str(rows)], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    for r in range(4):
        assert f"Passed {r}" in p.stdout, p.stdout
    got = [json.loads(line) for line in rows.read_text().splitlines()]
    assert len(got) == 1 and got[0]["pattern"] == "reduce_scatter" and got[0]["algo"] == "direct"
    assert got[0]["mismatches"] == 0 and got[0]["type"] == dtype and got[0]["op"] == op and got[0]["ranks"] == 4
