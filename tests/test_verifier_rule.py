"""The comparison rule of the halo checks without a GPU: the rule itself (tests/field_compare.py), the fields that need
it (a run into NaN, a run into signed zeros), and the fault table of tests/test_gpu_verifiers.py against the emulated
verifiers (tests/emu_device.py, tests/halo_dtype_emu.py), which count with the same rule as the kernels."""
import ctypes

import numpy as np
import pytest
import torch

from hpc_patterns_b200.models.halo import DTYPES, _native_type
from hpc_patterns_b200.ops.halo import stencil_step_reference
from tests.field_compare import count_far, count_wrong, same_bits
from tests.halo_dtype_emu import HaloDtypeEmu, typed_view
from tests.verifier_faults import (TYPES, assert_run_reaches, bits_of, lanes, other_nan, run_field, special_counts,
                                   special_step, ulp_away, value_faults, value_row)

IDS = {t: DTYPES[t] for t in TYPES}


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_rule_on_the_value_table(dtype):
    for name, want, got, counted in value_faults(dtype):
        assert count_wrong(got.reshape(1), want.reshape(1)) == counted, name
    nan = torch.tensor([float("nan")], dtype=dtype)
    assert same_bits(nan, other_nan(dtype).reshape(1)) and not torch.equal(nan, nan)
    zeros = torch.tensor([0.0, -0.0], dtype=dtype)
    assert torch.equal(zeros, zeros.flip(0)) and count_wrong(zeros, zeros.flip(0)) == 2


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_growing_run_into_nan_is_correct_under_the_rule(dtype):
    """alpha=0.3, s=0.7 (fp64: 3, 7): a correct field full of NaN, which `!=` and torch.equal call wrong."""
    for cp in (0, 1):
        field = run_field(2, 13, 1024, dtype, "grow", cp)[0]
        assert_run_reaches(field, "grow", cp)
        assert same_bits(field, field.clone())
        assert not torch.equal(field, field) and int((field != field).sum()) == special_counts(field)["nan"]


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_decaying_run_into_signed_zeros_is_checked_under_the_rule(dtype):
    """alpha = s = 0.1: the field passes through subnormals into ±0; a wrong sign of zero or a flushed subnormal, which
    `!=` and torch.equal accept, is wrong."""
    field = run_field(2, 13, 1024, dtype, "decay", 0)[0]
    assert_run_reaches(field, "decay", 0)
    d = field.double()
    flushed = torch.where((d != 0) & (d.abs() < torch.finfo(dtype).tiny), torch.zeros_like(field) * field.sign(), field)
    assert int((flushed != field).sum()) == count_wrong(flushed, field) > 0
    field = run_field(2, 13, 1024, dtype, "decay", 1)[0]
    assert_run_reaches(field, "decay", 1)
    flipped = -field
    assert torch.equal(flipped, field)
    assert count_wrong(flipped, field) == field.numel()


def test_count_far_is_the_allreduce_rule():
    assert count_far(np.array([13.0, 13.0 + 2.0 ** -20], dtype=np.float32), 13.0) == 0       # 1 ulp: within 1e-6
    assert count_far(np.array([np.nan, 12.0, 13.0 + 2.0 ** -19, 13.0]), 13.0) == 3
    assert count_far(torch.tensor([13.0, 13.0625], dtype=torch.bfloat16).double().numpy(), 13.0) == 1


# ------------------------------------------------------------------------------------ the emulated verifiers ----
class _Emu:
    def __init__(self):
        self.emu = HaloDtypeEmu()

    def put(self, t):
        t = t.contiguous()
        addr = self.emu.alloc(t.numel() * t.element_size())
        typed_view(addr, t.numel(), t.dtype).copy_(t.reshape(-1))
        return addr

    def count(self, call, *args, dtype):
        cnt = self.emu.alloc(8)
        getattr(self.emu, call)(*args, cnt, 0, **_native_type(dtype))
        return ctypes.c_int64.from_address(cnt).value

    def verify_step(self, new, old, up, dn, alpha, s):
        rows, n = old.shape
        return self.count("halo_verify_step", self.put(new), self.put(old), self.put(up), self.put(dn), rows, n,
                          alpha, s, dtype=old.dtype)

    def verify_init(self, u, rank, world, steps, alpha, s):
        rows, n = u.shape
        return self.count("halo_verify_from_init", self.put(u), rows, n, rank, world, steps, alpha, s, dtype=u.dtype)


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_emulated_verify_step_value_faults(dtype):
    emu = _Emu()
    n = 128
    want, got, expected, _ = value_row(dtype, n)
    z = torch.full((n,), -0.0, dtype=dtype)
    assert count_wrong(stencil_step_reference(want[None], z, z, 1.0, 1.0), want[None]) == 0
    assert emu.verify_step(want[None], want[None], z, z, 1.0, 1.0) == 0
    assert emu.verify_step(got[None], want[None], z, z, 1.0, 1.0) == expected > 0


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_emulated_verify_step_special_inputs(dtype):
    emu = _Emu()
    old, up, dn = special_step(dtype, 3, 256 * lanes(dtype))
    want = stencil_step_reference(old, up, dn, 0.5, 0.25)
    c = special_counts(want)
    assert c["nan"] and c["inf"] and c["-0"] and c["+0"] and c["subnormal"], c
    assert emu.verify_step(want, old, up, dn, 0.5, 0.25) == 0
    got = want.clone()
    bits_of(got).view(-1)[::7] ^= 1
    assert emu.verify_step(got, old, up, dn, 0.5, 0.25) == count_wrong(got, want) > 0


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
@pytest.mark.parametrize("run", ["grow", "decay"])
def test_emulated_verify_init_special_fields(dtype, run):
    emu = _Emu()
    world, rows, n = 2, 13, 256
    field, steps, alpha, s = run_field(world, rows, n, dtype, run, 0)
    want = field[rows:].contiguous()
    assert emu.verify_init(want, 1, world, steps, alpha, s) == 0
    got = want.clone()
    d = want.double()
    if run == "grow":
        i = torch.nonzero(torch.isnan(d).view(-1))[:, 0]
        got.view(-1)[i[0]] = 1.0                      # finite where NaN is due: counted
        got.view(-1)[i[1]] = other_nan(dtype)         # another NaN: not counted
    else:
        i = torch.nonzero(((d != 0) & (d.abs() < torch.finfo(dtype).tiny)).view(-1))[:, 0]
        got.view(-1)[i[0]] = 0.0 * torch.sign(got.view(-1)[i[0]])   # flushed subnormal: counted
    assert emu.verify_init(got, 1, world, steps, alpha, s) == 1


@pytest.mark.parametrize("dtype", TYPES, ids=IDS.get)
def test_emulated_verify_positions(dtype):
    emu = _Emu()
    rows, L = 3, lanes(dtype)
    n = 64 * L
    g = torch.Generator().manual_seed(3)
    ext = (torch.randint(-512, 513, (rows + 2, n), generator=g).float() / 16).to(dtype)
    old, up, dn = ext[1:-1].contiguous(), ext[0].contiguous(), ext[-1].contiguous()
    want = stencil_step_reference(old, up, dn)
    for where in ([(0, 0)], [(rows - 1, n - 1)], [(1, 5 * L + k) for k in range(L)], [(0, k) for k in range(32)]):
        got = want.clone()
        for r, c in where:
            got[r, c] = ulp_away(got[r, c])
        assert emu.verify_step(got, old, up, dn, 0.5, 0.25) == len(where)
    got = want.clone()
    bits_of(got).bitwise_xor_(1)
    assert emu.verify_step(got, old, up, dn, 0.5, 0.25) == rows * n


def test_emulated_count_mismatch_follows_the_device_rule():
    from tests.emu_device import EmuNative

    emu = EmuNative()
    v = np.full(64, 13.0, dtype=np.float32)
    v[3] = np.nextafter(np.float32(13.0), np.float32(14.0))    # 1 ulp off: within 1e-6, not counted
    v[5], v[9] = np.nan, 12.0
    cnt = ctypes.c_int64(0)
    emu.count_mismatch(v.ctypes.data, 64, 13.0, "float", ctypes.addressof(cnt), 0)
    assert cnt.value == 2
