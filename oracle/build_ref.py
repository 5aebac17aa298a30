"""Recipe for the reference binaries the comparison runs use: the upstream project's OpenMP concurrency bench.

argonne-lcf/HPC-Patterns' ``concurency/main.cpp`` + ``concurency/bench_omp.cpp`` build with plain ``g++ -fopenmp``
(target regions fall back to the host).  The one build-line addition is ``-Domp_target_alloc_host=omp_target_alloc``
(an Intel extension mapped to the standard call; the sources are compiled as they are, straight from the reference
checkout).  Two programs, one per mode, like the reference's own concurency/run_omp.sh:6-7:

    oracle/_ref/omp_nowait  oracle/_ref/omp_host_threads

The reference checkout is ``$HPCP_REFERENCE`` (default ``/root/reference``).  Without a readable checkout nothing is
built and nothing fails: whatever compares against the reference then reports it as unavailable or uses the stored
reference output under tests/golden/.  ``oracle/_ref/`` is git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from typing import Dict, Optional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.path.join(ROOT, "oracle", "_ref")
MODES = {"nowait": "NOWAIT", "host_threads": "HOST_THREADS"}


def reference_src() -> str:
    return os.environ.get("HPCP_REFERENCE", "/root/reference")


def host_cxx() -> str:
    return os.environ.get("HOSTCXX") or ("/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++") or "g++")


def binary(mode: str, out_dir: str = OUT_DIR) -> Optional[str]:
    """The built reference program for `mode`, or None."""
    exe = os.path.join(out_dir, f"omp_{mode}")
    return exe if mode in MODES and os.access(exe, os.X_OK) else None


def build(src: Optional[str] = None, out_dir: str = OUT_DIR) -> Dict[str, str]:
    """Compile both modes into `out_dir` (up to date: skipped).  Returns {mode: path} of what exists afterwards."""
    con = os.path.join(src or reference_src(), "concurency")
    srcs = [os.path.join(con, f) for f in ("main.cpp", "bench_omp.cpp")]
    if not all(os.access(s, os.R_OK) for s in srcs):
        print(f"oracle: no readable reference checkout at {os.path.dirname(con)}; reference binaries not built")
        return {}
    os.makedirs(out_dir, exist_ok=True)
    built = {}
    for mode, flag in MODES.items():
        exe = os.path.join(out_dir, f"omp_{mode}")
        if not (os.path.exists(exe) and all(os.path.getmtime(exe) >= os.path.getmtime(s) for s in srcs)):
            p = subprocess.run([host_cxx(), "-O2", "-std=c++17", "-fopenmp", f"-D{flag}",
                                "-Domp_target_alloc_host=omp_target_alloc", *srcs, "-o", exe],
                               capture_output=True, text=True, timeout=900)
            if p.returncode != 0:
                print(f"oracle: the reference's {mode} bench does not build: {p.stderr[-500:]}")
                continue
        built[mode] = exe
    return built


if __name__ == "__main__":
    print(build(sys.argv[1] if len(sys.argv) > 1 else None))
