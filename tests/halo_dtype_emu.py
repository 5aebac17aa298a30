"""The emulated device of tests/emu_device.py extended to K-halo fields of type double, bfloat16 and half.

``HaloDtypeEmu`` runs ``halo_stencil_ctas`` / ``halo_init`` / ``halo_stencil`` / ``halo_verify_from_init`` /
``halo_verify_step`` with the field-type contract of the kernels when a call names a type (``dtype=...``), and leaves
fp32 calls, which never name one, to ``EmuNative`` unchanged.  The arithmetic is ``reference_steps``'s: widen to the
compute type, one rounded operation at a time, round once to the field type.  ``calls`` records the field type of every
native halo call, so that the tests can check that fp32 calls keep their old shape.
"""
import ctypes

import torch

from hpc_patterns_b200.models.halo import compute_dtype, initial_field, reference_steps
from tests.emu_device import EmuNative, _u32
from tests.field_compare import count_wrong

TORCH = {"float": torch.float32, "double": torch.float64, "bfloat16": torch.bfloat16, "half": torch.float16}


def typed_view(ptr, n, dtype):
    esz = torch.empty(0, dtype=dtype).element_size()
    return torch.frombuffer((ctypes.c_uint8 * (n * esz)).from_address(ptr), dtype=torch.uint8).view(dtype)


def step_rows(up, u, dn, alpha, s):
    """One step of rows u with boundary rows up / dn in the kernels' arithmetic (u.dtype is the field type)."""
    ct = compute_dtype(u.dtype)
    ext = torch.cat([up[None], u, dn[None]], 0).to(ct)
    a = torch.tensor(alpha, dtype=torch.float32).to(ct)
    b = torch.tensor(s, dtype=torch.float32).to(ct)
    return (a * ext[1:-1] + b * (ext[:-2] + ext[2:])).to(u.dtype)


class HaloDtypeEmu(EmuNative):
    def __init__(self, ctas=3):
        super().__init__(ctas)
        self.calls = []

    def halo_stencil_ctas(self, row_elems, mode="pull", tune=None, device=0, **kw):
        self.calls.append(("halo_stencil_ctas", kw.get("dtype")))
        return super().halo_stencil_ctas(row_elems, mode, tune, device)

    def halo_init(self, u, halo_lo, halo_hi, rows, row_elems, rank, world, stream, **kw):
        self.calls.append(("halo_init", kw.get("dtype")))
        if "dtype" not in kw:
            return super().halo_init(u, halo_lo, halo_hi, rows, row_elems, rank, world, stream)
        dt = TORCH[kw["dtype"]]
        f = initial_field(world, rows, row_elems, dt)
        G, first = world * rows, rank * rows
        typed_view(u, rows * row_elems, dt).view(rows, row_elems).copy_(f[first:first + rows])
        if halo_lo:
            typed_view(halo_lo, row_elems, dt).copy_(f[(first + G - 1) % G])
        if halo_hi:
            typed_view(halo_hi, row_elems, dt).copy_(f[(first + rows) % G])

    def halo_stencil(self, a, mode="pull", tune=None, device=0, stream=0, **kw):
        self.calls.append(("halo_stencil", kw.get("dtype")))
        if "dtype" not in kw:
            return super().halo_stencil(a, mode, tune, device, stream)
        dt = TORCH[kw["dtype"]]
        esz = torch.empty(0, dtype=dt).element_size()
        tune = tune or {}
        R, n = a["rows"], a["row_elems"]
        assert (n * esz) % 16 == 0, "a row is a multiple of 16 bytes"
        tile = (tune.get("tile_kb") or 16) * 1024 // esz
        tiles = (n + tile - 1) // tile
        t0, t1 = a.get("tile_begin", 0), a.get("tile_end", 0) or tiles
        assert 0 <= t0 < t1 <= tiles, "bad column-tile range"
        c0, c1 = t0 * tile, min(n, t1 * tile)
        ctas = super().halo_stencil_ctas(n, mode, tune)
        fs = a.get("flag_set", 0)
        self.launches.append((mode, a["step_base"], a["steps"], t0, t1, fs))
        if mode != "none" and a["steps"] > 1 and not self.concurrent_ranks:
            assert a["left_u"][0] == a["u"][0] and a["right_u"][0] == a["u"][0]
        for g in range(a["step_base"], a["step_base"] + a["steps"]):
            i, o = g & 1, (g + 1) & 1
            if mode != "none":
                for c in range(ctas):
                    for side in (0, 1):
                        self._await(self._flag(a["flags_local"], fs, side, c), g,
                                    f"step {g}, word (set {fs}, side {side}, cta {c})")
            u_in = typed_view(a["u"][i], R * n, dt).view(R, n)
            u_out = typed_view(a["u"][o], R * n, dt).view(R, n)
            if mode == "pull":
                up = typed_view(a["left_u"][i], R * n, dt).view(R, n)[R - 1]
                dn = typed_view(a["right_u"][i], R * n, dt).view(R, n)[0]
            else:
                up, dn = typed_view(a["halo_lo"][i], n, dt), typed_view(a["halo_hi"][i], n, dt)
            new = step_rows(up[c0:c1], u_in[:, c0:c1], dn[c0:c1], a["alpha"], a["s"])
            u_out[:, c0:c1] = new
            if mode == "push":
                typed_view(a["left_halo_hi"][o], n, dt)[c0:c1] = new[0]
                typed_view(a["right_halo_lo"][o], n, dt)[c0:c1] = new[R - 1]
            if mode != "none":
                for c in range(ctas):
                    _u32(self._flag(a["flags_right"], fs, 0, c)).value = g + 1
                    _u32(self._flag(a["flags_left"], fs, 1, c)).value = g + 1
        return ctas

    def halo_verify_from_init(self, u, rows, row_elems, rank, world, steps, alpha, s, mismatch, stream, **kw):
        self.calls.append(("halo_verify_from_init", kw.get("dtype")))
        if "dtype" not in kw:
            return super().halo_verify_from_init(u, rows, row_elems, rank, world, steps, alpha, s, mismatch, stream)
        dt = TORCH[kw["dtype"]]
        want = reference_steps(initial_field(world, rows, row_elems, dt), steps, alpha, s)[rank * rows:(rank + 1) * rows]
        got = typed_view(u, rows * row_elems, dt).view(rows, row_elems)
        ctypes.c_int64.from_address(mismatch).value += count_wrong(got, want)

    def halo_verify_step(self, u_new, u_old, up_row, dn_row, rows, row_elems, alpha, s, mismatch, stream, **kw):
        self.calls.append(("halo_verify_step", kw.get("dtype")))
        if "dtype" not in kw:
            return super().halo_verify_step(u_new, u_old, up_row, dn_row, rows, row_elems, alpha, s, mismatch, stream)
        dt = TORCH[kw["dtype"]]
        old = typed_view(u_old, rows * row_elems, dt).view(rows, row_elems)
        want = step_rows(typed_view(up_row, row_elems, dt), old, typed_view(dn_row, row_elems, dt), alpha, s)
        got = typed_view(u_new, rows * row_elems, dt).view(rows, row_elems)
        ctypes.c_int64.from_address(mismatch).value += count_wrong(got, want)

