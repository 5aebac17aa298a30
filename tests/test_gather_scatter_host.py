"""The reduce-scatter and all-gather layers that run without a GPU: the Python refusals say the native launcher's
words and come before anything is allocated, the torch references agree with the exact owner-first oracle, the
constant-data check of ReduceScatterMiniapp tells every rank's result from the poison and from its neighbours', and the
JSON rows have their patterns."""
import types

import pytest
import torch

import hpc_patterns_b200
from hpc_patterns_b200.models.allreduce import (ReduceScatterMiniapp, ReduceScatterResult, rs_expected, rs_input,
                                                rs_poison)
from hpc_patterns_b200.models.alltoall import AllgatherMiniapp, AllgatherResult
from hpc_patterns_b200.ops.allreduce import check_reduce_scatter_args, reduce_scatter_reference
from hpc_patterns_b200.ops.alltoall import all_gather_reference, check_gather_args
from tests.reduce_scatter_oracle import bits_equal, expected, make_inputs

C = hpc_patterns_b200.native()


@pytest.mark.parametrize("world,n,dtype", [(4, 3, "float"), (4, 0, "float"), (17, 4, "float"), (0, 4, "int"),
                                           (4, 4, "half"), (2, 1, "double_int"), (16, 16, "uchar"), (3, 8, "short")])
def test_reduce_scatter_refusals_say_the_native_words(world, n, dtype):
    native_words = C.reduce_scatter_refusal(world, n, dtype, "maxloc" if dtype == "double_int" else "sum")
    if native_words:
        with pytest.raises(ValueError) as e:
            check_reduce_scatter_args(world, n, dtype)
        assert str(e.value) == native_words
    else:
        check_reduce_scatter_args(world, n, dtype)


@pytest.mark.parametrize("world,block", [(4, 8), (4, 0), (17, 16), (0, 16), (1, 16), (16, 48)])
def test_all_gather_refusals_say_the_native_words(world, block):
    native_words = C.all_gather_refusal(world, block)
    if native_words:
        with pytest.raises(ValueError) as e:
            check_gather_args(world, block)
        assert str(e.value) == native_words
    else:
        check_gather_args(world, block)


class _NoComm:
    """A communicator that fails if a refused miniapp touches it."""
    rank, world = 0, 4

    def __getattr__(self, name):
        raise AssertionError(f"comm.{name} used before the refusal")


@pytest.mark.parametrize("kw,words", [
    (dict(dtype="float", op="band"), "band reduces integer types only"),
    (dict(dtype="int", op="maxloc"), "maxloc reduces value-index pair types only"),
    (dict(dtype="2int", op="sum"), "sum reduces arithmetic types only"),
    (dict(dtype="int", op="bor", algo="nccl"), "nccl reduce-scatters sum, prod, min and max only"),
    (dict(dtype="uint", op="max", algo="nccl"), "compares uint as a signed torch type"),
    (dict(algo="ring"), "algo must be one of"),
])
def test_reduce_scatter_miniapp_refuses_before_allocating(kw, words):
    with pytest.raises(ValueError, match=words):
        ReduceScatterMiniapp(_NoComm(), 0, 10, **kw)


def test_allgather_miniapp_refuses_before_allocating():
    comm = types.SimpleNamespace(rank=0, world=4)
    with pytest.raises(ValueError, match="all-gather: block_bytes"):
        AllgatherMiniapp(comm, 0, 24)
    with pytest.raises(ValueError, match="algo must be one of"):
        AllgatherMiniapp(comm, 0, 16, "ring")


@pytest.mark.parametrize("world", [1, 2, 3, 5])
@pytest.mark.parametrize("dtype,op", [("float", "sum"), ("int", "sum"), ("bfloat16", "sum"), ("half", "prod"),
                                      ("int", "bxor"), ("uchar", "lor"), ("short", "max"), ("float_int", "maxloc"),
                                      ("2int", "minloc")])
def test_reference_is_the_owner_first_fold(dtype, op, world):
    n = 16
    sends = make_inputs(world, n, dtype, op, seed=3, launch=0)
    if dtype in ("float_int", "2int"):
        ts = [torch.frombuffer(bytearray(s), dtype=torch.uint8) for s in sends]
        ref = reduce_scatter_reference(ts, op, dtype)
        for r in range(world):
            want = expected(sends, r, op, dtype)
            if world == 1:
                assert bytes(ref[r].numpy().tobytes()) == want
            else:
                assert bits_equal(bytes(ref[r].numpy().tobytes()), want, dtype) == 0
        return
    ref = reduce_scatter_reference(sends, op, dtype)
    for r in range(world):
        assert bits_equal(ref[r], expected(sends, r, op, dtype), dtype) == 0, r


def test_all_gather_reference_is_the_concatenation():
    sends = [torch.arange(8, dtype=torch.float32) + 10 * p for p in range(3)]
    got = all_gather_reference(sends)
    assert got.shape == (3, 32) and torch.equal(got.view(torch.float32), torch.stack(sends))


@pytest.mark.parametrize("op", ["sum", "prod", "min", "max", "band", "bor", "bxor", "land", "lor", "lxor"])
def test_constant_data_check_tells_ranks_apart(op):
    """Every rank's expected value is exact in every type that takes the op, differs from the poison, and for the sum
    from the result of reducing any other segment."""
    for world in range(1, 17):
        for r in range(world):
            want = rs_expected(op, r, world)
            assert want != rs_poison(op, world), (op, world, r)
            if op == "sum":
                assert want == sum(rs_input(op, p, r, world) for p in range(world))
                assert want <= 232 and want == int(want)        # exact in uchar and in bfloat16's 8 bits
                others = {sum(rs_input(op, p, q, world) for p in range(world)) for q in range(world) if q % 8 != r % 8}
                assert want not in others


def test_json_rows():
    row = ReduceScatterResult("direct", "float", 4, 1 << 20, 0.5, 0, 4, "sum").row()
    assert row["pattern"] == "reduce_scatter" and row["mismatches"] == 0
    assert row["GBps_sent_per_rank"] == pytest.approx(3 * (1 << 20) * 4 / 0.5e-3 / 1e9)
    row = AllgatherResult("pull", 4, 1 << 20, 0.25, 0, 8).row()
    assert row["pattern"] == "allgather" and row["variant"] == "pull"
    assert row["GBps_sent_per_rank"] == pytest.approx(3 * (1 << 20) / 0.25e-3 / 1e9)


def test_front_door_lists_the_programs():
    import hpc_patterns_b200.__main__ as front

    assert "reduce_scatter" in front.__doc__ and "allgather" in front.__doc__
    assert "reduce_scatter" in front._GPU_PROGRAMS and "allgather" in front._GPU_PROGRAMS
