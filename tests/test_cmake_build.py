"""The CMake front end (↔ aurora.mpich.miniapps/src/CMakeLists.txt): configure, build every target for
sm_90a, and run the ctest cases that need no GPU (native unit tests, --cpu plumbing paths, host bench)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("cmake") is None or shutil.which("nvcc") is None, reason="needs cmake and nvcc")
def test_cmake_configure_build_and_host_ctest(tmp_path):
    env = dict(os.environ)
    env.pop("CXX", None)    # the image's CXX wrapper cannot link OpenMP (see Makefile)
    cfg = subprocess.run(["cmake", ROOT, "-DCMAKE_CXX_COMPILER=/usr/bin/g++", "-DCMAKE_CUDA_HOST_COMPILER=/usr/bin/g++"],
                         cwd=tmp_path, capture_output=True, text=True, env=env, timeout=600)
    assert cfg.returncode == 0, cfg.stdout[-3000:] + cfg.stderr[-3000:]
    jobs = str(max(2, os.cpu_count() or 2))
    bld = subprocess.run(["cmake", "--build", ".", "-j", jobs], cwd=tmp_path, capture_output=True, text=True, env=env,
                         timeout=1800)
    assert bld.returncode == 0, bld.stdout[-3000:] + bld.stderr[-3000:]
    for exe in ("concurency", "omp_con", "peer2pear", "topology", "allreduce.float", "allreduce.int",
                "interop_torchless", "interop_driver", "native_selftest",
                "allreduce-mpi-sycl.float", "allreduce-map-mpi-omp-offload.float", "peer2pear_i", "peer2pear_w",
                "sycl_con", "omp_nowait", "omp_host_threads"):          # incl. the reference's program names
        assert (tmp_path / exe).exists(), exe
    listing = subprocess.run(["ctest", "-N"], cwd=tmp_path, capture_output=True, text=True).stdout
    for case in ("allreduce.float", "allreduce.int.collective", "peer2pear.put", "peer2pear.sendrecv"):
        assert case in listing                       # the N-rank GPU cases are registered like upstream's
    t = subprocess.run(["ctest", "-R", "host|selftest", "--output-on-failure"], cwd=tmp_path, capture_output=True,
                       text=True, timeout=600)
    assert t.returncode == 0 and "100% tests passed" in t.stdout, t.stdout[-3000:]
