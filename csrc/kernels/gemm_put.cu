// K-gemm-put: bf16 GEMM on the Hopper tensor cores (wgmma) whose epilogue PUTs the result tile into a
// peer GPU over NVLink — "compute step followed by a transfer" as ONE kernel.
//
//     C[M,N] (fp32) = A[M,K] (bf16, K-major) . B[N,K]^T (bf16, K-major)
//     C is written to c_local and/or to c_peer (a peer-mapped pointer), then the arrival epoch is
//     published on the peer (same release/acquire protocol as every other kernel of the suite).
//
// Nothing in the reference is GEMM-shaped; this kernel is the tensor-core member of
// the suite's "fuse the transfer into the producing kernel" family, next to K-fused-triad-put
// (stream triad -> put) and K-ring (accumulate -> forward).  Stock comparison: cuBLAS GEMM followed
// by cudaMemcpyPeerAsync (two operations, the C tile goes to HBM and is read back before it moves).
//
// Structure (persistent, one CTA per SM, 384 threads, wgmma.cuh: gemm_persistent):
//   warp 0          TMA producer : cp.async.bulk.tensor.2d (SWIZZLE_128B) A[128x64] + B[256x64] per stage,
//                                  4-stage smem ring, full/empty mbarriers
//   warpgroups 1,2  consumers    : wgmma.mma_async m64n256k16 (64 rows each), fp32 accumulators in registers;
//                                  epilogue: registers -> padded smem staging -> 128-byte row segments
//                                  -> st.global to c_local and/or the peer (coalesced NVLink stores)
#include "api.h"

#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "wgmma.cuh"

namespace hpcp {

namespace {

using namespace umma;  // tile geometry, descriptors, TMA / wgmma wrappers, rasterisation, tensor-map encoder

constexpr int kStages = 4;
constexpr size_t kSmemBytes = gemm_smem_bytes<kStages>(0);

struct GemmDev {
  void* c_local;    // may be null; fp32 [M,N], or bf16 [M,N] when out_bf16
  void* c_peer;     // may be null
  int out_bf16;
  int m, n, k;
  int tiles_m, tiles_n;
  SyncOps sync;
};

// The kernel is the suite's persistent tile loop (wgmma.cuh: gemm_persistent) with this policy: grouped
// rasterisation over the whole C, stores (local and/or peer) in the epilogue, one arrival epoch at the end.
struct PutPolicy {
  static constexpr bool kHasAuxWarp = false;
  const GemmDev& g;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    tile_coords(tile, g.tiles_m, g.tiles_n, m_blk, n_blk);
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    epilogue_store_tile(g, d, epi_stage_buf(epi_smem, ew), m0, n0, ew, lane);
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  // Put epilogue: the last CTA publishes the arrival epoch on the peer.
  __device__ __forceinline__ void finish() const {
    if (g.sync.ticket != nullptr)
      last_cta_publish(g.sync.ticket, g.sync.ticket_base + gridDim.x, g.sync.signal_flag, g.sync.signal_epoch);
  }
};

// kCluster == 2: thread-block clusters of two CTAs working on vertically adjacent tiles that share the B tile
// (wgmma.cuh: gemm_persistent).
template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_put_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                    const __grid_constant__ GemmDev g) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, PutPolicy{g});
}

// Alternative epilogue (opt-in, `tma_epilogue`): the C tile leaves through the TMA unit — swizzled [32 x 128 B]
// pieces in shared memory, one cp.async.bulk.tensor.2d store (UTMASTG) per piece and destination — instead of
// 128-bit st.global from the epilogue warps.  Frees the LSU and sends the peer copy as bulk stores.
struct PutMaps {
  CUtensorMap c_local;  // valid iff g.c_local != nullptr
  CUtensorMap c_peer;   // valid iff g.c_peer != nullptr
};
struct PutTmaPolicy {
  static constexpr bool kHasAuxWarp = false;
  const GemmDev& g;
  const PutMaps& maps;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    tile_coords(tile, g.tiles_m, g.tiles_n, m_blk, n_blk);
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    epilogue_tma_tiles(g.out_bf16 != 0, d, epi_smem, ew, lane, [&](const unsigned char* tile, int col) {
      if (g.c_peer != nullptr) tma_store_2d(&maps.c_peer, n0 + col, m0 + ew * kEpiRows, tile);
      if (g.c_local != nullptr) tma_store_2d(&maps.c_local, n0 + col, m0 + ew * kEpiRows, tile);
    });
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  __device__ __forceinline__ void finish() const {
    epilogue_tma_drain();  // the bulk stores are performed before the arrival epoch is published
    if (g.sync.ticket != nullptr)
      last_cta_publish(g.sync.ticket, g.sync.ticket_base + gridDim.x, g.sync.signal_flag, g.sync.signal_epoch);
  }
};

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_put_tma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                        const __grid_constant__ GemmDev g, const __grid_constant__ PutMaps maps) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, PutTmaPolicy{g, maps});
}

}  // namespace

int launch_gemm_put(const void* a_bf16, const void* b_bf16, void* c_local, void* c_peer, int m, int n,
                    int k, bool out_bf16, const SyncOps& sync, int ctas, int device, cudaStream_t stream,
                    int cluster, bool tma_epilogue) {
  HPCP_REQUIRE(m > 0 && n > 0 && k > 0 && m % kBM == 0 && n % kBN == 0 && k % kBK == 0,
               "gemm_put: M, N, K must be multiples of 128, 256, 64");
  HPCP_REQUIRE(c_local != nullptr || c_peer != nullptr, "gemm_put: no output");
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(a_bf16) & 15) == 0 && (reinterpret_cast<uintptr_t>(b_bf16) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(c_local) & 15) == 0 && (reinterpret_cast<uintptr_t>(c_peer) & 15) == 0,
               "gemm_put: pointers must be 16-byte aligned");
  HPCP_REQUIRE(sync.signal_flag == nullptr || sync.ticket != nullptr, "gemm_put: a signal needs a ticket counter");
  // Cluster mode needs an even number of tile rows per raster group (pairs share n_blk).
  HPCP_REQUIRE(cluster >= 0 && cluster <= 2, "gemm_put: cluster must be 0 (auto), 1 or 2");
  const bool pairable = (m / kBM) % 2 == 0 && ((m / kBM) % kGroupM) % 2 == 0;
  HPCP_REQUIRE(cluster != 2 || pairable, "gemm_put: cluster=2 needs an even number of 128-row tiles per raster group");
  const bool use_cluster = cluster != 1 && pairable;
  const CUtensorMap map_a = make_kmajor_map(a_bf16, m, k, kBM);
  const CUtensorMap map_b = make_kmajor_map(b_bf16, n, k, use_cluster ? kBN / 2 : kBN);
  GemmDev g{};
  g.c_local = c_local;
  g.c_peer = c_peer;
  g.out_bf16 = out_bf16 ? 1 : 0;
  g.m = m;
  g.n = n;
  g.k = k;
  g.tiles_m = m / kBM;
  g.tiles_n = n / kBN;
  g.sync = sync;
  const int tiles = g.tiles_m * g.tiles_n;
  const int sms = device_sm_count(device);
  int grid = std::min(tiles, ctas > 0 ? ctas : sms);
  if (tma_epilogue) {
    PutMaps maps{};
    if (c_local != nullptr) maps.c_local = make_c_tile_map(c_local, m, n, out_bf16);
    if (c_peer != nullptr) maps.c_peer = make_c_tile_map(c_peer, m, n, out_bf16);
    constexpr size_t smem_t = gemm_smem_bytes<kStages>(kTmaEpiSmemBytes - kEpiWarps * kEpiWarpBytes);
    static_assert(smem_t + 1024 <= 227 * 1024, "GEMM stages + two store tiles per epilogue warp must fit in 227 KiB");
    if (!use_cluster || grid < 2) {
      const CUtensorMap map_b_full = use_cluster ? make_kmajor_map(b_bf16, n, k, kBN) : map_b;
      HPCP_ENABLE_SMEM(gemm_put_tma_kernel<1>, smem_t);
      gemm_put_tma_kernel<1><<<grid, kThreads, smem_t, stream>>>(map_a, map_b_full, g, maps);
      HPCP_CUDA(cudaGetLastError());
      return grid;
    }
    grid &= ~1;
    HPCP_ENABLE_SMEM(gemm_put_tma_kernel<2>, smem_t);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(grid));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_t;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    HPCP_CUDA(cudaLaunchKernelEx(&cfg, gemm_put_tma_kernel<2>, map_a, map_b, g, maps));
    return grid;
  }
  if (!use_cluster || grid < 2) {
    const CUtensorMap map_b_full = use_cluster ? make_kmajor_map(b_bf16, n, k, kBN) : map_b;
    HPCP_ENABLE_SMEM(gemm_put_kernel<1>, kSmemBytes);
    gemm_put_kernel<1><<<grid, kThreads, kSmemBytes, stream>>>(map_a, map_b_full, g);
    HPCP_CUDA(cudaGetLastError());
    return grid;
  }
  grid &= ~1;  // whole pairs
  HPCP_ENABLE_SMEM(gemm_put_kernel<2>, kSmemBytes);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(grid));
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  HPCP_CUDA(cudaLaunchKernelEx(&cfg, gemm_put_kernel<2>, map_a, map_b, g));
  return grid;
}

}  // namespace hpcp
