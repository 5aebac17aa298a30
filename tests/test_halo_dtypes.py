"""K-halo's field types on the CPU: double, bfloat16 and half next to float.

1. ``initial_field`` / ``reference_steps`` (the PyTorch contract the GPU tests compare against) equal an independent
   numpy implementation bit for bit; numpy has no bfloat16, so its round-to-nearest-even is done on uint32 bit patterns.
2. The tests' data notice the faults a typed kernel could have: 16-bit values carried in fp32 across steps, truncation
   instead of RNE, contraction to FMA, bf16 bits read as fp16, double computed in fp32, one lane pair swapped in a
   16-byte vector, subnormals flushed.
3. ``bin/halo --cpu --type T --dump`` and ``bin/halo.T --cpu`` equal ``reference_steps``; a bad ``--type`` is a usage
   error.
4. The Python layer (HaloStencil / VirtualRing / step_from_host / stock steps / stencil_step checks) on the emulated
   device of tests/halo_dtype_emu.py; fp32 calls into the native module keep their old shape.
5. No double, bfloat16 or half instantiation of the K-halo stencil kernel touches local memory.
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from hpc_patterns_b200.models import halo as halo_mod
from hpc_patterns_b200.models.halo import initial_field, reference_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = {"float": torch.float32, "double": torch.float64, "bfloat16": torch.bfloat16, "half": torch.float16}
COEFFS = [(0.5, 0.25), (0.3, 0.7)]


# ---------------------------------------------------------------------------------------- numpy oracle ----
def np_u0(world, rows, n):
    g = np.arange(world * rows, dtype=np.uint64)[:, None]
    j = np.arange(n, dtype=np.uint64)[None, :]
    h = ((g * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) ^ ((j * np.uint64(40503) + (j >> np.uint64(11)))
                                                                   & np.uint64(0xFFFFFFFF))
    return ((h & np.uint64(0xFFFF)).astype(np.int64) - 32768).astype(np.float32) * np.float32(1.0 / 1024.0)


def bf16_rne(x32, trunc=False):
    """fp32 -> bf16 bits (uint16): round-to-nearest-even (or truncation) on the bit pattern; no NaNs in this data."""
    b = np.ascontiguousarray(x32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    if not trunc:
        b = b + np.uint64(0x7FFF) + ((b >> np.uint64(16)) & np.uint64(1))
    return (b >> np.uint64(16)).astype(np.uint16)


def bf16_widen(bits):
    return (bits.astype(np.uint32) << np.uint32(16)).view(np.float32)


def half_trunc(x32):
    h = x32.astype(np.float16)
    over = np.abs(h.astype(np.float32)) > np.abs(x32)
    return np.where(over, np.nextafter(h, np.float16(0)), h)


class Oracle:
    """One type's storage <-> compute conversions and step, with optional faults."""

    def __init__(self, name, fault=None):
        self.name, self.fault = name, fault

    def store(self, x):                     # compute -> storage (numpy array of the storage representation)
        if self.name == "bfloat16":
            return bf16_rne(x, trunc=self.fault == "trunc")
        if self.name == "half":
            return half_trunc(x) if self.fault == "trunc" else x.astype(np.float16)
        if self.name == "double":
            return x.astype(np.float64)
        return x.astype(np.float32)

    def widen(self, v):
        if self.name == "bfloat16":
            if self.fault == "bf16_as_fp16":
                return v.view(np.float16).astype(np.float32)
            return bf16_widen(v)
        if self.name == "half":
            return v.astype(np.float32)
        return v

    def compute_type(self):
        return np.float64 if self.name == "double" and self.fault != "double_in_fp32" else np.float32

    def step(self, w, alpha, s):
        ct = self.compute_type()
        w = w.astype(ct)
        a, b = ct(np.float32(alpha)), ct(np.float32(s))
        side = (b * (np.roll(w, 1, 0) + np.roll(w, -1, 0))).astype(ct)
        if self.fault == "fma":            # alpha*u + side with one rounding (exact product, fp64 sum, one fp32 round)
            return (np.float64(a) * w.astype(np.float64) + side.astype(np.float64)).astype(ct)
        return (a * w).astype(ct) + side

    def run(self, world, rows, n, steps, alpha, s, start=None):
        """Returns the field after `steps` steps in the compute type (values of the storage type)."""
        v = self.store(np_u0(world, rows, n) if start is None else start)
        if self.fault == "carry" and self.name in ("bfloat16", "half"):
            w = self.widen(v)
            for _ in range(steps):
                w = self.step(w, alpha, s)
            return self.widen(self.store(w)).astype(np.float64)
        for _ in range(steps):
            w = self.step(self.widen(v), alpha, s)
            if self.fault == "flush":
                tiny = np.float32(torch.finfo(TYPES[self.name]).smallest_normal)
                w = np.where(np.abs(w) < tiny, np.float32(0), w).astype(w.dtype)
            v = self.store(w)
            if self.fault == "swap_pair":  # the first two lanes (double) / 32-bit pairs of every 16-byte vector swap
                raw = v.view(np.uint32).reshape(v.shape[0], -1, 4).copy()
                order = [2, 3, 0, 1] if self.name == "double" else [1, 0, 2, 3]
                raw = raw[:, :, order]
                v = np.ascontiguousarray(raw).reshape(v.shape[0], -1).view(v.dtype)
        return self.widen(v).astype(np.float64)


def torch_f64(t):
    return t.double().numpy()


@pytest.mark.parametrize("name", list(TYPES))
@pytest.mark.parametrize("alpha,s", COEFFS)
def test_reference_equals_numpy_oracle(name, alpha, s):
    dt = TYPES[name]
    f = initial_field(3, 2, 1024, dt)
    assert f.dtype == dt
    assert np.array_equal(torch_f64(f), Oracle(name).run(3, 2, 1024, 0, alpha, s))
    got = reference_steps(f, 6, alpha, s)
    assert got.dtype == dt and np.array_equal(torch_f64(got), Oracle(name).run(3, 2, 1024, 6, alpha, s))
    if name == "bfloat16":   # the bit-pattern RNE is the one torch uses, on ties too
        x = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 ** -130 * 3], dtype=torch.float32)
        assert np.array_equal(bf16_rne(x.numpy()), x.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16))


def test_reference_of_float32_is_unchanged():
    """fp32 callers see the same expression as before the field types existed."""
    f = initial_field(2, 3, 512)
    u = f.clone()
    a, b = torch.tensor(0.3), torch.tensor(0.7)
    for _ in range(4):
        u = a * u + b * (torch.roll(u, 1, 0) + torch.roll(u, -1, 0))
    assert torch.equal(reference_steps(f, 4, 0.3, 0.7), u)


FAULTS = [("bfloat16", "carry"), ("half", "carry"), ("bfloat16", "trunc"), ("half", "trunc"), ("float", "fma"),
          ("bfloat16", "fma"), ("half", "fma"), ("bfloat16", "bf16_as_fp16"), ("double", "double_in_fp32"),
          ("double", "swap_pair"), ("bfloat16", "swap_pair"), ("half", "swap_pair")]


@pytest.mark.parametrize("name,fault", FAULTS)
def test_faults_are_reported(name, fault):
    """Each fault, run on the data of the tests (three ranks of two rows, 0.3 / 0.7), changes the field."""
    world, rows, n, steps = 3, 2, 1 << 16, 5
    want = torch_f64(reference_steps(initial_field(world, rows, n, TYPES[name]), steps, 0.3, 0.7))
    assert np.array_equal(want, Oracle(name).run(world, rows, n, steps, 0.3, 0.7))
    assert not np.array_equal(want, Oracle(name, fault).run(world, rows, n, steps, 0.3, 0.7))


@pytest.mark.parametrize("name", ["bfloat16", "half"])
def test_flushed_subnormals_are_reported(name):
    """Fields a few steps above the smallest subnormal: reference_steps keeps subnormal results, a flush is caught."""
    dt = TYPES[name]
    tiny = torch.finfo(dt).smallest_normal
    g = torch.Generator().manual_seed(3)
    f = (torch.randint(-64, 65, (6, 4096), generator=g).double() * (tiny / 64)).to(dt)
    want = reference_steps(f, 3, 0.3, 0.7)
    assert int(((want != 0) & (want.abs() < tiny)).sum()) > 1000
    start = f.float().numpy()
    assert np.array_equal(torch_f64(want), Oracle(name).run(0, 0, 0, 3, 0.3, 0.7, start=start))
    assert not np.array_equal(torch_f64(want), Oracle(name, "flush").run(0, 0, 0, 3, 0.3, 0.7, start=start))


# ------------------------------------------------------------------------------------- native --cpu ----
DUMP = {"float": np.float32, "double": np.float64, "half": np.float16, "bfloat16": np.uint16}


def _dump_tensor(path, name, shape):
    raw = np.fromfile(path, dtype=DUMP[name]).reshape(shape)
    t = torch.from_numpy(raw.view(np.int16) if name == "bfloat16" else raw)
    return t.view(torch.bfloat16) if name == "bfloat16" else t


@pytest.mark.parametrize("name", list(TYPES))
@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("ranks", [1, 2, 3])
@pytest.mark.parametrize("rows", [1, 2, 5])
@pytest.mark.parametrize("by", ["option", "program"])
def test_native_host_path(bin_dir, tmp_path, name, mode, ranks, rows, by):
    dump, row_bytes, steps, iters, warmup = tmp_path / "field.raw", 1040, 3, 2, 1
    prog = ["halo", "--type", name] if by == "option" else [f"halo.{name}"]
    p = subprocess.run([os.path.join(bin_dir, prog[0]), *prog[1:], "--cpu", "-n", str(ranks), "--rows", str(rows),
                        "--bytes", str(row_bytes), "--steps", str(steps), "--iters", str(iters), "--warmup",
                        str(warmup), "--mode", mode, "--dump", str(dump)], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stdout + p.stderr
    assert p.stdout.count("Passed") == ranks and f"type={name} |" in p.stdout
    dt = TYPES[name]
    n = row_bytes // torch.empty(0, dtype=dt).element_size()
    got = _dump_tensor(dump, name, (ranks * rows, n))
    want = reference_steps(initial_field(ranks, rows, n, dt), steps * (iters + warmup))
    assert torch.equal(got, want)


@pytest.mark.parametrize("bad", ["int", "fp8", "quad"])
def test_native_bad_type_is_a_usage_error(bin_dir, bad):
    p = subprocess.run([os.path.join(bin_dir, "halo"), "--cpu", "--type", bad], capture_output=True, text=True)
    assert p.returncode == 1 and "Usage: halo" in p.stdout and "--type" in p.stderr


def test_native_json_row_has_the_type(bin_dir, tmp_path):
    out = tmp_path / "rows.jsonl"
    p = subprocess.run([os.path.join(bin_dir, "halo.half"), "--cpu", "-n", "2", "--bytes", "64", "--steps", "2",
                        "--json", str(out)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    import json
    row = json.loads(out.read_text().splitlines()[-1])
    assert row["type"] == "half" and row["pattern"] == "halo" and row["mismatches"] == 0


# ----------------------------------------------------------------------------- Python layer, emulated ----
@pytest.fixture
def emu(monkeypatch):
    from tests.emu_device import install
    from tests.halo_dtype_emu import HaloDtypeEmu

    e = HaloDtypeEmu()
    install(monkeypatch.setattr, e)
    return e


@pytest.mark.parametrize("name", list(TYPES))
@pytest.mark.parametrize("mode", ["pull", "push"])
@pytest.mark.parametrize("world,rows", [(1, 1), (2, 3), (3, 2), (5, 4)])
def test_virtual_ring(emu, name, mode, world, rows):
    dt = TYPES[name]
    ring = halo_mod.VirtualRing(world, 5000 - 5000 % 16 + 16, rows, mode, devices=[0] * world, tune={"tile_kb": 1},
                                dtype=dt)
    ring.step(2)
    ring.step(1, persistent=world == 1)
    n = ring.ranks[0].row_elems
    got = ring.gather()
    assert got.dtype == dt and torch.equal(got, reference_steps(initial_field(world, rows, n, dt), 3))
    for hs in ring.ranks:
        assert hs.verify_from_init() == 0 and hs.verify_last_step() == 0
    ring.close()
    kinds = {k for k, _ in emu.calls}
    assert kinds == {"halo_stencil_ctas", "halo_init", "halo_stencil", "halo_verify_from_init", "halo_verify_step"}
    assert {t for _, t in emu.calls} == {None if name == "float" else name}   # fp32 calls name no type


@pytest.mark.parametrize("name", list(TYPES))
def test_stock_steps_and_host_steps(emu, name):
    dt = TYPES[name]
    ring = halo_mod.VirtualRing(1, 2048, 2, "pull", devices=[0], tune={"tile_kb": 1}, dtype=dt)
    hs = ring.ranks[0]
    for _ in range(3):
        hs.stock_step("memcpy")
    assert torch.equal(hs.u_tensor(), reference_steps(initial_field(1, 2, hs.row_elems, dt), 3))
    assert hs.verify_last_step() == 0
    ring.close()
    ring = halo_mod.VirtualRing(2, 3 * 1024 + 32, 3, "push", devices=[0, 0], tune={"tile_kb": 1}, dtype=dt)
    bufs = [hs.make_host_buffers() for hs in ring.ranks]
    assert bufs[0][0].dtype == dt
    for k in range(3):
        for hs, b in zip(ring.ranks, bufs):
            hs.step_from_host(b[k & 1], b[(k + 1) & 1], chunks=3)
    got = torch.cat([b[1] for b in bufs], 0)
    assert torch.equal(got, reference_steps(initial_field(2, 3, ring.ranks[0].row_elems, dt), 3))
    ring.close()


def test_unsupported_dtype_is_refused(emu):
    with pytest.raises(ValueError, match="dtype"):
        halo_mod.VirtualRing(1, 2048, 2, "pull", devices=[0], dtype=torch.int32)


# ------------------------------------------------------------------------------------------- SASS ----
def test_non_float_stencil_kernels_use_no_local_memory(native):
    obj = os.path.join(ROOT, "build", "kernels", "halo_stencil.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    fns = re.split(r"\n\s+Function : ", sass)[1:]
    # the nine non-float instantiations; the fp32 pull kernel keeps a documented once-per-tile local slot
    typed = [f for f in fns if re.search(r"halo_stencil_kernelI(?!f)", f.split("\n", 1)[0])]
    assert len(typed) == 9
    for f in typed:
        assert not re.search(r"\b(STL|LDL)", f), f.split("\n", 1)[0]
