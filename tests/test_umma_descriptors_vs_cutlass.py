"""The hand-built wgmma shared-memory matrix descriptor (csrc/kernels/wgmma.cuh: make_smem_desc) and the 128-byte
swizzle the TMA epilogues write by hand, against CUTLASS's definitions of the same (headers vendored in the image under
flashinfer/data/cutlass/include; skipped when absent)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROGRAM = r"""
#include "kernels/wgmma.cuh"   // first: it needs the driver-API typedefs before CUTLASS pulls in its own CUDA headers
#include <cstdio>
#include <cute/tensor.hpp>
#include <cute/arch/mma_sm90_desc.hpp>
using namespace cute;
int main() {
  // The 128-byte swizzle the TMA epilogues write by hand (wgmma.cuh: epilogue_tma_tiles: chunk c of row r at
  // c ^ (r % 8)) against CUTLASS's Swizzle<3,4,3>, the layout a SWIZZLE_128B tensor map reads / writes.
  int bad = 0;
  for (int r = 0; r < 32; ++r)
    for (int c = 0; c < 8; ++c)
      bad += int(Swizzle<3, 4, 3>{}(r * 128 + c * 16)) != r * 128 + ((c ^ (r & 7)) << 4);
  printf("swizzle_mismatches %d\n", bad);
  // Shared-memory matrix descriptor (K-major, SWIZZLE_128B, 8-row x 128-byte atoms every 1024 bytes) against
  // CUTLASS's bit-field definition of the wgmma descriptor.
  int bad_desc = 0;
  for (uint32_t addr : {0x0u, 0x400u, 0xC000u, 0x2A400u, 0x38C00u}) {
    GmmaDescriptor d;
    d.bitfield.start_address_ = uint16_t((addr & 0x3FFFF) >> 4);
    d.bitfield.leading_byte_offset_ = 1;
    d.bitfield.stride_byte_offset_ = 1024 >> 4;
    d.bitfield.base_offset_ = 0;
    d.bitfield.layout_type_ = uint8_t(SM90::GMMA::LayoutType::B128);
    bad_desc += d.desc_ != hpcp::umma::make_smem_desc(addr);
  }
  printf("smem_desc_mismatches %d\n", bad_desc);
  return 0;
}
"""


def _cutlass_include():
    import importlib.util

    spec = importlib.util.find_spec("flashinfer")          # located, not imported
    if spec is None or not spec.submodule_search_locations:
        return None
    d = os.path.join(list(spec.submodule_search_locations)[0], "data", "cutlass", "include")
    return d if os.path.exists(os.path.join(d, "cute", "arch", "mma_sm90_desc.hpp")) else None


def test_instruction_descriptor_matches_cutlass(tmp_path):
    inc = _cutlass_include()
    if inc is None:
        pytest.skip("no vendored CUTLASS headers in this image")
    src = tmp_path / "desc.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "desc"
    p = subprocess.run(["nvcc", "-ccbin", "/usr/bin/g++", "-std=c++17", "--expt-relaxed-constexpr", "-I", inc, "-I",
                        os.path.join(ROOT, "csrc"), "-gencode", "arch=compute_90a,code=sm_90a", str(src), "-o",
                        str(exe)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-2000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60).stdout
    assert "swizzle_mismatches 0" in out and "smem_desc_mismatches 0" in out, out
