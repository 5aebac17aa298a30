"""In-tree build of the native extension ``hpc_patterns_b200/_C*.so``.

``python -m hpc_patterns_b200._build`` (or ``make ext``) compiles every CUDA
source for sm_90a (``-gencode arch=compute_90a,code=sm_90a -lineinfo``) into
``build/libhpcp.a`` through the Makefile, compiles the pybind11 bindings and links
the extension next to this file, so the ``.so`` travels with a repo snapshot.
The reference has no Python build at all (its builds are the shell one-liners
``concurency/run_sycl.sh:6`` / ``p2p/run.sh:3-5`` and a CMake project).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"]


def host_cxx() -> str:
    # The image exports CXX=/opt/gcc/bin/g++ (a wrapper that cannot link OpenMP).
    return os.environ.get("HOSTCXX") or ("/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++")


def ext_path() -> Path:
    return ROOT / "hpc_patterns_b200" / ("_C" + sysconfig.get_config_var("EXT_SUFFIX"))


def run(cmd: list[str]) -> None:
    print("+", " ".join(cmd), flush=True)
    subprocess.run(cmd, cwd=ROOT, check=True)


def build(jobs: int | None = None, cli: bool = True) -> Path:
    import pybind11

    jobs = jobs or max(2, os.cpu_count() or 2)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    targets = ["build/libhpcp.a"] + (["cli"] if cli else [])
    run(["make", f"-j{jobs}", f"NVCC={nvcc}", f"HOSTCXX={host_cxx()}"] + targets)

    out = ext_path()
    obj = ROOT / "build" / "bindings.o"
    src = ROOT / "csrc" / "bindings.cpp"
    deps = [src, ROOT / "build" / "libhpcp.a"] + list((ROOT / "csrc").rglob("*.h*"))
    if out.exists() and all(out.stat().st_mtime >= d.stat().st_mtime for d in deps):
        print(f"up to date: {out}")
        return out
    includes = [f"-I{sysconfig.get_paths()['include']}", f"-I{pybind11.get_include()}",
                f"-I{ROOT / 'csrc'}", "-I/usr/local/cuda/include"]
    run([host_cxx(), "-O2", "-std=c++17", "-fPIC", "-fopenmp", "-fvisibility=hidden", *includes,
         "-c", str(src), "-o", str(obj)])
    run([nvcc, "-ccbin", host_cxx(), *ARCH_FLAGS, "-shared", "-Xcompiler", "-fPIC",
         str(obj), str(ROOT / "build" / "libhpcp.a"), "-o", str(out), "-lgomp", "-ldl"])
    return out


if __name__ == "__main__":
    build(cli="--no-cli" not in sys.argv)
