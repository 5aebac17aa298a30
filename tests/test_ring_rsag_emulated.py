"""The allreduce miniapp's ``--algo ring-rsag`` on the CPU: its byte and slot accounting, and the Python twin as 2 and 4
``gloo`` processes on the emulated device (tests/emu_device.py with tests/rsag_emu.py, harness of
tests/test_multiprocess_emulated.py), whose ``ring_rsag`` awaits and publishes the kernel's arrival words hop by hop."""
import pytest

import tests.test_multiprocess_emulated as mp_harness
from hpc_patterns_b200.models import allreduce as ar

_HARNESS_WORKER = mp_harness._worker


def _rsag_worker(*args):
    """The harness's worker, with the emulated device that also runs ring_rsag."""
    from tests.rsag_emu import use_in_worker

    use_in_worker()
    _HARNESS_WORKER(*args)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_bytes_and_slots(world):
    nbytes = world * (1 << 20)
    assert ar.bytes_sent_per_rank("ring-rsag", nbytes, world) == 2 * nbytes * (world - 1) / world
    assert ar.bytes_sent_per_rank("ring", nbytes, world) == nbytes * (world - 1)
    assert ar.bytes_sent_per_rank("twoshot", nbytes, world) == nbytes * (world - 1) / world
    assert ar.rsag_layout(nbytes, 9, world) == (9, nbytes // world * max(world - 1, 1))
    assert ar.ring_layout(nbytes, 9, world, 0) == (9, nbytes * max(world - 1, 1))
    assert ar.ring_layout(nbytes, 9, world, 2) == (18, 2 * nbytes)


def test_eight_ranks_default_size():
    """P = 8 at the default 2^25 floats: 224 MiB sent per rank instead of the fused ring's 896 MiB, 112 MiB of slots
    instead of 896 MiB."""
    nbytes = 4 << 25
    assert ar.bytes_sent_per_rank("ring-rsag", nbytes, 8) == 224 << 20
    assert ar.bytes_sent_per_rank("ring", nbytes, 8) == 896 << 20
    assert ar.rsag_layout(nbytes, 0, 8)[1] == 112 << 20


def test_row_reports_the_rsag_bytes():
    r = ar.AllreduceResult("ring-rsag", "float", 4, 1 << 20, 2.0, 0, 4)
    assert r.row()["GBps_sent_per_rank"] == pytest.approx(2 * 3 / 4 * (4 << 20) / 2e-3 / 1e9)
    assert "ring-rsag" in ar.ALGOS and "ring-rsag" in ar.VIRTUAL_ALGOS


@pytest.mark.parametrize("world,port", [(2, 29791), (4, 29792)])
def test_allreduce_python_twin_ring_rsag(world, port, monkeypatch):
    monkeypatch.setattr(mp_harness, "_worker", _rsag_worker)
    res = mp_harness._run(world, port, "allreduce", "ring-rsag")
    for rank, r in res.items():
        assert r["leaked"] == 0
        for x in r["results"]:
            assert x["mismatches"] == 0 and x["passed"], (rank, x)
            assert x["launches"] == 3                      # one warm-up + two timed launches, one kernel each
