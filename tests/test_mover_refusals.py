"""Host-side refusals of the data movers' launchers: each bad call must be refused with its own message before the
launcher's first CUDA call.

The calls run in one child process that sees no CUDA device (``CUDA_VISIBLE_DEVICES=""``), so no pointer below is ever
dereferenced: a refusal that fired late, or not at all, ends in the CUDA error of the first runtime call instead of
the expected message, and a misaligned vector access can never reach a GPU.  The addresses are fake.
"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = 1 << 24          # a 16-byte aligned (fake) address; BASE + 4 is only 4-byte aligned

ALIGN = "pointers must be 16-byte aligned"
TRIAD_ARGS = ("a_local", "a_peer", "b", "c")


def _triad(n=4096, n_put=0, engine="ldst", off=None, a_peer=BASE + 0x100000):
    ptrs = {"a_local": BASE, "a_peer": a_peer, "b": BASE + 0x200000, "c": BASE + 0x300000}
    if off is not None:
        ptrs[off] += 4
    return ["triad_put", ptrs["a_local"], ptrs["a_peer"], ptrs["b"], ptrs["c"], 3.0, n, engine, n_put]


def _fused(kind, off, engine):
    if kind == "triad":
        cmd = {"kind": "triad", "n": 4096, "a": BASE, "b": BASE + 0x100000, "c": BASE + 0x200000}
    else:
        cmd = {"kind": "copy", "n": 4096, "dst": BASE, "src": BASE + 0x100000}
    cmd[off] += 4
    return ["fused_bench", [{"kind": "busy", "n": 64, "tripcount": 1, "a": BASE + 0x300000}, cmd], engine]


CASES = {}
for _e in ("ldst", "tma"):
    CASES[f"n=0-{_e}"] = (_triad(n=0, engine=_e), "triad_put: n must be positive")
    CASES[f"n=0-no-put-{_e}"] = (_triad(n=0, engine=_e, a_peer=0), "triad_put: n must be positive")
    for _p in TRIAD_ARGS:
        CASES[f"{_p}+4-{_e}"] = (_triad(engine=_e, off=_p), "triad_put: " + ALIGN)
    CASES[f"a_local+4-no-put-{_e}"] = (_triad(engine=_e, off="a_local", a_peer=0), "triad_put: " + ALIGN)
    for _p in ("a", "b", "c"):
        CASES[f"fused-triad-{_p}+4-{_e}"] = (_fused("triad", _p, _e), "fused bench: triad " + ALIGN)
    for _p in ("dst", "src"):
        CASES[f"fused-copy-{_p}+4-{_e}"] = (_fused("copy", _p, _e), "fused bench: copy " + ALIGN)
    CASES[f"n%4-{_e}"] = (_triad(n=4094, engine=_e), "triad_put: n must be a multiple of 4 elements")
    CASES[f"n%n_put-{_e}"] = (_triad(n=12288, n_put=8192, engine=_e), "triad_put: n must be a multiple of n_put")
# Halo mode: the halo must be whole 16 KiB tiles (LdSt) or whole TMA stages (here 16 KiB, the default).
CASES["halo-not-tile-ldst"] = (_triad(n=3 * 2048, n_put=2048, engine="ldst"),
                               "triad_put: halo (n_put) must be a multiple of 16 KiB")
CASES["halo-not-tile-tma"] = (_triad(n=3 * 6144, n_put=6144, engine="tma"),
                              "triad_put: halo (n_put) must be a multiple of the TMA tile size")

CHILD = r"""
import json, sys
import hpc_patterns_b200
C = hpc_patterns_b200.native()
out = {}
for name, call in json.loads(sys.stdin.read()).items():
    try:
        if call[0] == "triad_put":
            _, al, ap, b, c, s, n, engine, n_put = call
            C.triad_put(al, ap, b, c, s, n, engine, {}, {}, 0, 0, 0, 0, n_put)
        else:
            _, cmds, engine = call
            C.fused_bench(cmds, engine, {}, 0, 0)
        out[name] = "no error"
    except Exception as e:
        out[name] = f"{type(e).__name__}: {e}"
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def refusals(native):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    p = subprocess.run([sys.executable, "-c", CHILD], input=json.dumps({k: v[0] for k, v in CASES.items()}),
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=300)
    assert p.returncode == 0, p.stderr
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(CASES))
def test_refused_before_any_cuda_call(refusals, case):
    want = CASES[case][1]
    got = refusals[case]
    assert got.startswith("RuntimeError: " + want), got
