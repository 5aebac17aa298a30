"""Argument validation of the fused collective GEMMs — runs without a GPU (every check fires before any CUDA call)."""
import pytest
import torch

import hpc_patterns_b200
from hpc_patterns_b200.ops.gemm import allgather_gemm, gemm_all_to_all, gemm_put, gemm_reduce_scatter


def _bf16(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_python_wrappers_reject_bad_operands():
    with pytest.raises(TypeError):
        gemm_reduce_scatter(torch.zeros(256, 64), _bf16(256, 64), [0, 0], 0)
    with pytest.raises(ValueError, match="multiples"):
        gemm_reduce_scatter(_bf16(128, 64), _bf16(256, 64), [0, 0], 0)          # M not a multiple of 128 * world
    with pytest.raises(ValueError, match="shard"):
        gemm_reduce_scatter(_bf16(256, 64), _bf16(256, 64), [torch.zeros(64, 256), torch.zeros(128, 256)], 0)
    with pytest.raises(ValueError, match="c must be"):
        allgather_gemm(_bf16(256, 64), [0, 0], _bf16(256, 64), torch.zeros(256, 128), 0)
    with pytest.raises(ValueError, match="ready"):
        allgather_gemm(_bf16(256, 64), [0, 0], _bf16(256, 64), torch.zeros(256, 256), 0,
                       ready=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError, match="activation"):
        allgather_gemm(_bf16(256, 64), [0, 0], _bf16(256, 64), torch.zeros(256, 256), 0, activation="tanh")
    with pytest.raises(ValueError, match="receive buffer"):
        gemm_all_to_all(_bf16(256, 64), _bf16(256, 64), [torch.zeros(2, 128, 128), torch.zeros(2, 128, 256)], 0)
    with pytest.raises(TypeError):
        gemm_all_to_all(_bf16(256, 64), _bf16(256, 64), [0, 0], 0, out_dtype=torch.float16)
    # a tensor c_peer of the wrong type or size would be written past its end
    with pytest.raises(ValueError, match="c_peer"):
        gemm_put(_bf16(128, 64), _bf16(256, 64), None, _bf16(128, 256))                 # bf16, out_dtype fp32
    with pytest.raises(ValueError, match="c_peer"):
        gemm_put(_bf16(128, 64), _bf16(256, 64), None, torch.zeros(128, 256), out_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="c_peer"):
        gemm_put(_bf16(256, 64), _bf16(256, 64), torch.zeros(256, 256), torch.zeros(128, 256))
    # a short or mistyped a_src row block would be read past its end
    with pytest.raises(ValueError, match="a_src"):
        allgather_gemm(_bf16(256, 64), [_bf16(128, 64), _bf16(64, 64)], _bf16(256, 64), torch.zeros(256, 256), 0)
    with pytest.raises(ValueError, match="a_src"):
        allgather_gemm(_bf16(256, 64), [_bf16(128, 64), torch.zeros(128, 64)], _bf16(256, 64),
                       torch.zeros(256, 256), 0)


def test_native_launchers_reject_bad_shapes_and_modes():
    C = hpc_patterns_b200.native()
    with pytest.raises(RuntimeError, match="multiple of 128 \\* world"):
        C.gemm_reduce_scatter(16, 16, [16, 16, 16], m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="cluster"):
        C.gemm_reduce_scatter(16, 16, [16, 16], m=256, n=256, k=64, cluster=7)
    with pytest.raises(RuntimeError, match="even number of tile rows"):
        C.gemm_reduce_scatter(16, 16, [16, 16], m=256, n=256, k=64, cluster=2)   # one tile row per shard
    with pytest.raises(RuntimeError, match="shard pointer"):
        C.gemm_reduce_scatter(16, 16, [16, 0], m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="ticket"):
        C.gemm_reduce_scatter(16, 16, [16, 16], done_flags=[16, 16], m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="chunk_bytes"):
        C.allgather_gemm(128, [128, 128], 16, 16, ready=16, chunk_bytes=3000, m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="arrival counters"):
        C.allgather_gemm(128, [128, 128], 16, 16, m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="row block pointer"):
        C.allgather_gemm(128, [0, 0], 16, 16, ready=16, rank=0, m=256, n=256, k=64)
    with pytest.raises(RuntimeError, match="receive buffer"):
        C.gemm_all_to_all(16, 16, [16, 0], m=256, n=256, k=64)
    with pytest.raises((RuntimeError, ValueError)):
        C.gemm_all_to_all(16, 16, [], m=256, n=256, k=64)
    assert C.allgather_gemm_chunks_per_block(64, 0) == 4 and C.allgather_gemm_chunks_per_block(8192, 2048) == 1024


def test_ring_rejects_inconsistent_slot_policy():
    C = hpc_patterns_b200.native()
    with pytest.raises(RuntimeError, match="n_slots"):
        C.ring_allreduce(16, 16, 16, 16, 16, 16, world=8, n=1024, n_slots=3)
    with pytest.raises(RuntimeError, match="ack words"):
        C.ring_allreduce(16, 16, 16, 16, 16, 16, world=8, n=1024, n_slots=2)
    with pytest.raises(RuntimeError, match="left neighbour"):
        C.ring_allreduce(16, 16, 16, 16, 16, 16, world=4, n=1024, pull=True)
    with pytest.raises(RuntimeError, match="ack words"):
        C.ring_allreduce(16, 16, 16, 16, 16, 16, world=8, n=1024, n_slots=2, pull=True, va_left=16, slots_left=16)


def test_epilogue_activations_match_their_pytorch_twins_on_the_cpu():
    from hpc_patterns_b200.models.tensor_parallel import apply_activation
    from hpc_patterns_b200.ops.gemm import ACTIVATIONS

    x = torch.linspace(-4, 4, 33)
    assert ACTIVATIONS[0] == "none" and torch.equal(apply_activation(x, "none"), x)
    assert torch.equal(apply_activation(x, "relu"), x.clamp(min=0))
    t = torch.tanh(0.7978845608 * (x + 0.044715 * x ** 3))          # the formula the kernel evaluates
    assert torch.allclose(apply_activation(x, "gelu"), 0.5 * x * (1 + t), atol=1e-6)
    assert torch.allclose(apply_activation(x, "silu"), x / (1 + torch.exp(-x)), atol=1e-6)
    with pytest.raises(ValueError):
        apply_activation(x, "tanh")


def test_python_wrappers_marshal_arguments_the_way_the_extension_expects(monkeypatch):
    """No GPU here, so the launch itself fails — but it must fail INSIDE the native launcher (RuntimeError: no driver /
    tensor-map encoder), not at the pybind boundary (TypeError: wrong number / order / type of arguments)."""
    import hpc_patterns_b200
    from hpc_patterns_b200.ops import gemm as G

    real = hpc_patterns_b200.native()

    class Proxy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            return lambda *a, **k: fn(*[0 if x is None else x for x in a], **k)   # CPU tensors have device index None

    monkeypatch.setattr(G, "native", lambda: Proxy())
    monkeypatch.setattr(G, "current_stream", lambda dev: 0)
    a, b = _bf16(512, 128), _bf16(256, 128)
    calls = [
        lambda: G.gemm_put(a, b, torch.zeros(512, 256), 0),
        lambda: G.gemm_put(a, b, torch.zeros(512, 256, dtype=torch.bfloat16), 16, out_dtype=torch.bfloat16, cluster=2,
                           epilogue="tma", sync={"ticket": 16, "ticket_base": 3}),
        lambda: G.gemm_reduce_scatter(a, b, [torch.zeros(256, 256), torch.zeros(256, 256)], 1, done_flags=[16, 32],
                                      done_epoch=2, ticket=16, ticket_base=4, epilogue="tma"),
        lambda: G.gemm_reduce_scatter(a, b, [16, 32], 0, out_dtype=torch.bfloat16, cluster=1),
        lambda: G.gemm_reduce_scatter(a, b, [0, 0], 0, c_multicast=4096),
        lambda: G.gemm_all_to_all(a, b, [torch.zeros(2, 256, 256), torch.zeros(2, 256, 256)], 0, done_flags=[16, 32],
                                  ticket=16),
        lambda: G.allgather_gemm(a, [a[:256], a[256:]], b, torch.zeros(512, 256), 0,
                                 ready=torch.zeros(4, dtype=torch.int32), ready_base=8, chunk_bytes=2048,
                                 done_flags=[16, 32], done_epoch=1, ticket=16, timeout_ns=10, status=16,
                                 activation="silu"),
    ]
    for call in calls:
        with pytest.raises(RuntimeError):
            call()
