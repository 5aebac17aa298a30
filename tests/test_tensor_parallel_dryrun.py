"""Dry run of the tensor-parallel model classes on the CPU: the GPU-facing pieces (symmetric buffers, signal pads, the
native extension, the fused ops) are replaced by recorders, so that every line of the orchestration code — epochs,
tickets, flag addresses, launch counts, argument names — executes and can be checked without a device."""
import inspect
import types

import pytest
import torch

import hpc_patterns_b200
from hpc_patterns_b200.models import tensor_parallel as tp
from hpc_patterns_b200.ops import gemm as real_ops


class FakeComm:
    def __init__(self, rank, world):
        self.rank, self.world, self.local_rank = rank, world, rank
        self.device = 0          # Comm.device: the ordinal the rank->device mapping chose


class FakeSymmetricBuffer:
    base = 1 << 20

    def __init__(self, comm, nbytes, device, zero=True):
        FakeSymmetricBuffer.base += 1 << 24
        self.nbytes, self.rank, self.world = int(nbytes), comm.rank, comm.world
        self.ptrs = [FakeSymmetricBuffer.base + r * (1 << 20) for r in range(comm.world)]
        self.local_ptr = self.ptrs[comm.rank]
        self._t = torch.zeros(self.nbytes, dtype=torch.uint8)
        self.closed = False

    def tensor(self, dtype=torch.uint8):
        return self._t.view(dtype)

    def close(self):
        self.closed = True


class Recorder:
    """Stands in for the native module: constants come from the real one, every call is recorded."""

    def __init__(self):
        self.real = hpc_patterns_b200.native()
        self.calls = []

    def __getattr__(self, name):
        attr = getattr(self.real, name)
        if not callable(attr) or name == "allgather_gemm_chunks_per_block":
            return attr

        def call(*a, **k):
            self.calls.append((name, a, k))
            return 0
        return call


@pytest.fixture
def fakes(monkeypatch):
    rec = Recorder()
    op_calls = []

    def fake_op(name, ctas):
        real = getattr(real_ops, name)

        def op(*a, **k):
            inspect.signature(real).bind(*a, **k)          # unknown / missing argument names fail here
            op_calls.append((name, a, k))
            return ctas
        return op

    class Pads:
        def __init__(self, comm, device, extra_words=0, timeout_s=20.0):
            self.rank, self.world = comm.rank, comm.world
            self.timeout_ns, self.ticket_issued, self.barriers, self.closed = int(timeout_s * 1e9), 0, 0, False
            self.ticket_ptr, self.status_ptr = 777000, 778000

        def word(self, rank, index):
            return 900000 + rank * 4096 + 4 * index

        def advance_tickets(self, ctas):
            self.ticket_issued += ctas

        def device_barrier(self, stream):
            self.barriers += 1

        def check(self):
            pass

        def close(self):
            self.closed = True

    shim = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
    shim.empty = lambda *a, device=None, **k: torch.empty(*a, **k)
    shim.zeros = lambda *a, device=None, **k: torch.zeros(*a, **k)
    monkeypatch.setattr(tp, "torch", shim)
    monkeypatch.setattr(tp, "native", lambda: rec)
    monkeypatch.setattr(tp, "SymmetricBuffer", FakeSymmetricBuffer)
    monkeypatch.setattr(tp, "SignalPads", Pads)
    monkeypatch.setattr(tp, "gemm_reduce_scatter", fake_op("gemm_reduce_scatter", 148))
    monkeypatch.setattr(tp, "allgather_gemm", fake_op("allgather_gemm", 146))
    monkeypatch.setattr(tp._FusedLinearBase, "_stream", property(lambda self: 4242))
    return rec, op_calls


def test_row_parallel_orchestration(fakes):
    rec, ops = fakes
    C = rec.real
    layer = tp.RowParallelLinear(FakeComm(1, 4), 0, m=2048, n=512, k_local=256, epilogue="tma")
    assert tuple(layer.y.shape) == (512, 512) and layer.y.dtype == torch.float32
    x = torch.zeros(2048, 256, dtype=torch.bfloat16)
    for step in (1, 2):
        y = layer.forward(x)
        assert y is layer.y and layer.pads.barriers == step and layer.pads.ticket_issued == 148 * step
        name, a, k = ops[-1]
        assert name == "gemm_reduce_scatter" and a[3] == 1 and a[2] == layer.shard.ptrs
        assert k["done_epoch"] == step and k["ticket_base"] == 148 * (step - 1) and k["epilogue"] == "tma"
        assert k["done_flags"] == [layer.pads.word(q, C.PAD_DONE + 1) for q in range(4)]   # my slot on every rank
        memset, wait = rec.calls[-2], rec.calls[-1]
        assert memset[0] == "memset_async" and memset[1][:3] == (layer.y.data_ptr(), 0, 512 * 512 * 4)
        assert wait[0] == "wait_flags" and wait[1][:3] == (layer.pads.word(1, C.PAD_DONE), 4, step)
    assert layer.launches == 6
    layer.close()
    assert layer.shard.closed and layer.pads.closed
    bf = tp.RowParallelLinear(FakeComm(0, 2), 0, m=512, n=256, k_local=64, out_dtype=torch.bfloat16)
    bf.forward(torch.zeros(512, 64, dtype=torch.bfloat16))
    assert bf.y.dtype == torch.bfloat16 and rec.calls[-2][1][2] == 256 * 256 * 2 and ops[-1][2]["out_dtype"] == torch.bfloat16
    with pytest.raises(ValueError):
        tp.RowParallelLinear(FakeComm(0, 2), 0, m=512, n=256, k_local=64, reduce="all", out_dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        tp.RowParallelLinear(FakeComm(0, 3), 0, m=512, n=256, k_local=64)                  # 512 % (128 * 3) != 0


def test_column_parallel_orchestration(fakes):
    rec, ops = fakes
    C = rec.real
    layer = tp.ColumnParallelLinear(FakeComm(2, 4), 0, m=2048, n_local=256, k=512, out_dtype=torch.bfloat16,
                                    chunk_bytes=2048, activation="gelu")
    rows = 512
    assert layer.x_local.data_ptr() == layer.a_full.data_ptr() + 2 * rows * 512 * 2      # my rows inside the gathered A
    per_launch = C.allgather_gemm_chunks_per_block(512, 2048)
    x = torch.ones(rows, 512, dtype=torch.bfloat16)
    for step in (1, 2, 3):
        n_calls = len(rec.calls)
        y = layer.forward(x)
        assert y is layer.y and tuple(y.shape) == (2048, 256)
        name, a, k = ops[-1]
        assert name == "allgather_gemm" and a[4] == 2
        assert a[1] == [layer.a.ptrs[q] + q * rows * 512 * 2 for q in range(4)]            # rank q's row block on rank q
        assert k["ready_base"] == (step - 1) * per_launch and k["chunk_bytes"] == 2048 and k["activation"] == "gelu"
        assert k["done_epoch"] == step and k["ticket_base"] == 146 * (step - 1)
        waits = [c for c in rec.calls[n_calls:] if c[0] == "wait_flags"]
        if step == 1:
            assert not waits                                  # nothing to wait for before the first step
        else:                                                 # the peers' "done reading" epochs of the previous step
            assert waits[0][1][:3] == (layer.pads.word(2, C.PAD_DONE), 4, step - 1)
        assert bool((layer.x_local == 1).all()) and layer.pads.barriers == step
    layer.forward(None)                                       # rows written in place: no wait, no copy
    assert ops[-1][2]["done_epoch"] == 4
    layer.close()
    assert layer.a.closed


def test_parallel_mlp_chains_the_layers(fakes):
    rec, ops = fakes
    mlp = tp.ParallelMLP(FakeComm(0, 2), 0, tokens=512, hidden=256, ffn=1024, activation="silu")
    assert tuple(mlp.up.w.shape) == (512, 256) and tuple(mlp.down.w.shape) == (256, 512)
    out = mlp.forward(torch.zeros(256, 256, dtype=torch.bfloat16))
    assert tuple(out.shape) == (256, 256)
    (n1, a1, k1), (n2, a2, k2) = ops[-2:]
    assert n1 == "allgather_gemm" and k1["activation"] == "silu" and n2 == "gemm_reduce_scatter"
    assert a2[0] is mlp.up.y                                   # the hidden activations feed the second GEMM in place
    assert mlp.launches == mlp.up.launches + mlp.down.launches > 0
    mlp.close()


def test_layers_take_buffers_from_the_caller(fakes):
    """``_shared``: the buffers of virtual ranks made by a LocalGroup are used as given, nothing else is allocated;
    ParallelMLP hands its ``ctas`` and ``_shared`` parts to both layers."""
    rec, ops = fakes
    comm = FakeComm(1, 2)
    pads = [tp.SignalPads(comm, 0) for _ in range(4)]
    shard = FakeSymmetricBuffer(comm, 256 * 512 * 4, 0)
    a = FakeSymmetricBuffer(comm, 512 * 256 * 2, 0)
    before = FakeSymmetricBuffer.base
    row = tp.RowParallelLinear(comm, 0, m=512, n=512, k_local=64, _shared={"pads": pads[0], "shard": shard})
    col = tp.ColumnParallelLinear(comm, 0, m=512, n_local=256, k=256, _shared={"pads": pads[1], "a": a})
    assert FakeSymmetricBuffer.base == before
    assert row.pads is pads[0] and row.shard is shard and row.y.data_ptr() == shard.tensor().data_ptr()
    assert col.pads is pads[1] and col.a is a and col.a_full.data_ptr() == a.tensor().data_ptr()
    row.forward(torch.zeros(512, 64, dtype=torch.bfloat16))
    assert ops[-1][1][2] == shard.ptrs and pads[0].ticket_issued == 148
    col.forward(torch.zeros(256, 256, dtype=torch.bfloat16))
    assert ops[-1][1][1] == [a.ptrs[q] + q * 256 * 256 * 2 for q in range(2)] and pads[1].ticket_issued == 146
    with pytest.raises(ValueError):                              # a shard of the wrong size
        tp.RowParallelLinear(comm, 0, m=512, n=256, k_local=64, _shared={"pads": pads[0], "shard": shard})
    with pytest.raises(ValueError):
        tp.RowParallelLinear(comm, 0, m=512, n=512, k_local=64, reduce="all", _shared={"pads": pads[0], "shard": shard})
    up_a = FakeSymmetricBuffer(comm, 512 * 256 * 2, 0)
    down_shard = FakeSymmetricBuffer(comm, 256 * 256 * 4, 0)
    before = FakeSymmetricBuffer.base
    mlp = tp.ParallelMLP(comm, 0, tokens=512, hidden=256, ffn=512, activation="relu", ctas=6,
                         _shared={"up": {"pads": pads[2], "a": up_a}, "down": {"pads": pads[3], "shard": down_shard}})
    assert FakeSymmetricBuffer.base == before
    assert mlp.up.pads is pads[2] and mlp.up.a is up_a and mlp.down.pads is pads[3] and mlp.down.shard is down_shard
    mlp.forward(torch.zeros(256, 256, dtype=torch.bfloat16))
    assert [(name, k["ctas"]) for name, _, k in ops[-2:]] == [("allgather_gemm", 6), ("gemm_reduce_scatter", 6)]
    plain = tp.ParallelMLP(comm, 0, tokens=512, hidden=256, ffn=512)           # without: own buffers, every SM
    assert FakeSymmetricBuffer.base > before and plain.up.ctas == plain.down.ctas == 0


def test_tp_program_end_to_end_dry(fakes, monkeypatch, capsys):
    """`python -m hpc_patterns_b200 tp --check --mlp ...` with every GPU-facing piece replaced: the whole program
    (argument handling, the three layers, the MLP block, the JSON line) runs; the numbers mean nothing."""
    import json

    rec, ops = fakes
    shim = tp.torch

    class Event:
        def __init__(self, enable_timing=False):
            pass

        def record(self, *a):
            pass

        def elapsed_time(self, other):
            return 1.0

    shim.cuda = types.SimpleNamespace(is_available=lambda: True, device_count=lambda: 8, set_device=lambda d: None,
                                      synchronize=lambda d=None: None, Event=Event,
                                      current_stream=lambda d=None: types.SimpleNamespace(cuda_stream=0))
    shim.device = lambda kind, index=0: torch.device("cpu")
    shim.Generator = lambda device=None: torch.Generator()
    shim.randint = lambda lo, hi, shape, device=None, generator=None: torch.randint(lo, hi, shape, generator=generator)

    class Comm(FakeComm):
        def __init__(self):
            super().__init__(0, 1)

        def barrier(self):
            pass

        def max(self, v):
            return v

        def min(self, v):
            return v

        def close(self):
            pass

    monkeypatch.setattr(tp, "Comm", Comm)
    # the stock twins run for real on the CPU (world = 1: plain matmuls)
    rc = tp.main(["--check", "--mlp", "--tokens", "256", "--out-features", "512", "--in-features", "256", "--steps", "1",
                  "--rs-epilogue", "tma", "--chunk", "1024", "--cluster", "1"])
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert out["ranks"] == 1 and (out["m"], out["n"], out["k"]) == (256, 512, 256) and out["rs_epilogue"] == "tma"
    for key in ("row_parallel", "column_parallel", "mlp"):
        assert {"fused_ms", "stock_ms", "speedup"} <= set(out[key])
    assert "row_parallel_exact" in out and "column_parallel_exact" in out and "mlp_max_abs_diff" in out
    assert isinstance(out["mlp_within_bound"], bool) and isinstance(out["mlp_hidden_exact"], bool)   # judged
    assert rc in (0, 1)                                          # the recorders compute nothing, so 'exact' is false
    assert [name for name, _, _ in ops].count("allgather_gemm") >= 3
