// K-tc-busy: the tensor-core compute command `T` of the concurrency benchmark.
//
// The reference's compute command is a dependent-FMA chain on the general-purpose
// ALUs (concurency/bench.hpp:23-31).  On H100 most of the machine's compute capacity is the
// tensor cores, so the suite also offers a compute command that keeps the *tensor pipe*
// busy while copies run next to it: a per-CTA bf16 GEMM tile
//        D[128 x 256] (fp32, registers) += A[128 x 64] . B[256 x 64]^T        x tripcount
// * A and B tiles are fetched ONCE by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B)
//   into shared memory, completion on an mbarrier;
// * two warpgroups issue wgmma.mma_async m64n256k16 (64 rows each, 4 x K=16 per pass over
//   the 64-deep tile, `tripcount` passes), accumulating in registers;
// * each thread stores its accumulator fragment, so the result is checkable:
//   D = tripcount * (A . B^T), exact in fp32 for the small-integer operands used.
// The loop touches no global memory, so its duration is proportional to tripcount —
// the same property the FMA chain has — but the busy unit is the tensor core.
#include "api.h"

#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <mutex>

#include "../common/cuda_check.h"
#include "../common/ptx.cuh"
#include "wgmma.cuh"

namespace hpcp {

namespace {

constexpr int kTileM = 128;
constexpr int kTileN = 256;
constexpr int kTileK = 64;   // one 128-byte swizzle atom of bf16
constexpr int kThreads = 256;
constexpr uint32_t kABytes = kTileM * kTileK * 2;  // 16 KiB
constexpr uint32_t kBBytes = kTileN * kTileK * 2;  // 32 KiB

// Descriptors, TMA tensor loads and wgmma wrappers: wgmma.cuh (shared with the GEMM kernels).
using umma::cluster_cta_rank;
using umma::cluster_sync_all;
using umma::kAccRegs;
using umma::tma_load_2d;
using umma::tma_load_2d_multicast;

// Dynamic smem (1024-aligned): A tile | B tile ; static smem: the operand barrier.
// kCluster == 2: launched as thread-block clusters of two CTAs that share the B tile — each CTA
// fetches half of B (128 of its 256 rows) and TMA-multicasts it into both CTAs' shared memory.
template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    tc_busy_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                   float* __restrict__ out, uint32_t tripcount) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ __align__(8) uint64_t full_bar;

  // SWIZZLE_128B operand tiles must start on a 1024-byte boundary of the shared window.
  unsigned char* smem_a = smem + ((1024u - (ptx::smem_u32(smem) & 1023u)) & 1023u);
  unsigned char* smem_b = smem_a + kABytes;
  const int wg = threadIdx.x >> 7;              // warpgroup: accumulator rows [64 wg, 64 wg + 64)
  const int warp = (threadIdx.x >> 5) & 3;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    ptx::mbar_init(&full_bar, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // The peer CTA's mbarrier must be initialised before anything is multicast into it.
  if (kCluster > 1) cluster_sync_all();

  if (threadIdx.x == 0) {  // TMA producer: both operand tiles, once
    ptx::mbar_arrive_expect_tx(&full_bar, kABytes + kBBytes);
    tma_load_2d(smem_a, &map_a, 0, 0, &full_bar);
    if (kCluster > 1) {
      const uint32_t r = cluster_cta_rank();  // my half of B, delivered to both CTAs
      tma_load_2d_multicast(smem_b + r * (kBBytes / 2), &map_b, 0, static_cast<int>(r) * (kTileN / 2), &full_bar,
                            static_cast<uint16_t>(0x3));
    } else {
      tma_load_2d(smem_b, &map_b, 0, 0, &full_bar);
    }
  }
  ptx::mbar_wait(&full_bar, 0);  // operands landed in smem

  float d[kAccRegs] = {};  // tripcount 0 stores zeros
  const uint32_t sa = ptx::smem_u32(smem_a) + static_cast<uint32_t>(wg) * (kABytes / 2);
  const uint32_t sb = ptx::smem_u32(smem_b);
  for (uint32_t it = 0; it < tripcount; ++it) {
    umma::wgmma_fence_operand(d);
    umma::wgmma_fence();
    umma::wgmma_kblock(d, sa, sb, it != 0);
    umma::wgmma_commit();
    umma::wgmma_wait<1>();  // one pass in flight behind the one being issued
    umma::wgmma_fence_operand(d);
  }
  umma::wgmma_wait<0>();
  umma::wgmma_fence_operand(d);

  // Fragment -> row-major out[cta][128][256] (wgmma.cuh: fragment layout of wgmma_m64n256k16_bf16).
  const int row = wg * 64 + warp * 16 + (lane >> 2);
  float* out_tile = out + static_cast<size_t>(blockIdx.x) * kTileM * kTileN;
#pragma unroll
  for (int j = 0; j < kTileN / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
    *reinterpret_cast<float2*>(out_tile + static_cast<size_t>(row) * kTileN + col) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(out_tile + static_cast<size_t>(row + 8) * kTileN + col) =
        make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
  // Neither CTA of a pair may retire while the other could still be receiving its multicast.
  if (kCluster > 1) cluster_sync_all();
}

__global__ void tc_fill_operands_kernel(__nv_bfloat16* a, __nv_bfloat16* b) {
  // Small integers: every product and every partial sum is exact in bf16 / fp32.
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kTileN * kTileK; i += gridDim.x * blockDim.x) {
    const int r = i / kTileK, k = i % kTileK;
    if (r < kTileM) a[i] = __float2bfloat16(static_cast<float>((r + k) % 3 - 1));
    b[i] = __float2bfloat16(static_cast<float>((r * 2 + k) % 5 - 2));
  }
}

CUtensorMap make_operand_map(const void* base, int rows, int box_rows) {
  CUtensorMap map;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(kTileK), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(kTileK) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kTileK), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult r = umma::gemm_tensor_map_encoder()(
      &map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box,
      elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
      CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HPCP_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " + std::to_string(r));
  return map;
}

}  // namespace

size_t tc_busy_operand_bytes() { return static_cast<size_t>(kTileM + kTileN) * kTileK * 2; }
size_t tc_busy_out_elems_per_cta() { return static_cast<size_t>(kTileM) * kTileN; }

void launch_tc_fill_operands(void* operands, cudaStream_t stream) {
  __nv_bfloat16* a = static_cast<__nv_bfloat16*>(operands);
  tc_fill_operands_kernel<<<32, 256, 0, stream>>>(a, a + kTileM * kTileK);
  HPCP_CUDA(cudaGetLastError());
}

void launch_tc_busy(const void* operands, float* out, int ctas, uint32_t tripcount,
                    cudaStream_t stream, int cluster) {
  HPCP_REQUIRE(ctas >= 1, "tc_busy: need at least one CTA");
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(operands) & 127) == 0, "tc_busy: operands must be 128-byte aligned");
  HPCP_REQUIRE(cluster == 1 || cluster == 2, "tc_busy: cluster size must be 1 or 2");
  if (cluster == 2 && ctas % 2 != 0) cluster = 1;  // pairs only
  const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(operands);
  const CUtensorMap map_a = make_operand_map(a, kTileM, kTileM);
  const size_t smem = kABytes + kBBytes + 1024;  // slack for the 1024-byte alignment
  if (cluster == 1) {
    const CUtensorMap map_b = make_operand_map(a + kTileM * kTileK, kTileN, kTileN);
    HPCP_ENABLE_SMEM(tc_busy_kernel<1>, smem);
    tc_busy_kernel<1><<<ctas, kThreads, smem, stream>>>(map_a, map_b, out, tripcount);
    HPCP_CUDA(cudaGetLastError());
    return;
  }
  // Thread-block clusters of 2: each CTA loads and multicasts one half (128 rows) of B.
  const CUtensorMap map_b = make_operand_map(a + kTileM * kTileK, kTileN, kTileN / 2);
  HPCP_ENABLE_SMEM(tc_busy_kernel<2>, smem);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(ctas));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  HPCP_CUDA(cudaLaunchKernelEx(&cfg, tc_busy_kernel<2>, map_a, map_b, out, tripcount));
}

}  // namespace hpcp
