// K-gemm-rs and K-ag-gemm: the two tensor-parallel "GEMM next to a collective" steps as ONE kernel each.
//
//   GEMM -> reduce-scatter   every rank holds a K-slice: C_r = A_r[M,K_r] . B_r[N,K_r]^T is a partial sum of the
//   (K-gemm-rs)              whole C; rank q owns rows [q*M/P, (q+1)*M/P) of the sum.  The epilogue of a tile
//                            does not store: it ADDS the accumulator into the owner's fp32 shard over NVLink
//                            (red.global.add.v4.f32, 128-byte row segments), tile by tile while the tensor cores
//                            work on the next tile.  When a rank's last tile is out it publishes its arrival
//                            epoch on every owner.  Stock pattern: cuBLAS GEMM, then ncclReduceScatter.
//
//   GEMM -> all-reduce       same partial products, but every rank wants the whole sum: the epilogue issues
//   (K-gemm-ar, NVLS)        multimem.red.add.v4.f32 on the multicast mapping of C, the NVSwitch adds the segment
//                            into all P copies.  M*N*4 bytes leave each GPU once (a ring reduce-scatter +
//                            all-gather moves 2(P-1)/P of that and needs two passes).  Stock: cuBLAS + ncclAllReduce.
//
//   GEMM -> all-to-all       row block q of C_r = A_r . B_r^T belongs to rank q (expert outputs going home, a
//   (K-gemm-a2a)             Ulysses head/sequence swap): the epilogue stores every tile straight into slot r of
//                            rank q's receive buffer [P, M/P, N] over NVLink.  Stock: cuBLAS + ncclAllToAll.
//
//   all-gather -> GEMM       every rank holds a row block A_r[M/P,K] and needs C = A[M,K] . B_r[N,K]^T.  Warp 3
//   (K-ag-gemm)              of every CTA (idle in a plain GEMM) is a gather engine: TMA bulk copies pull 4 KiB
//                            pieces of the peers' row blocks over NVLink through a small smem ring into the
//                            local gathered A and count arrivals per 128-row block; the TMA producer of a tile
//                            waits for its block's count, so the GEMM starts on the local block at t = 0 and
//                            the transfer of block i+1 hides behind the math of block i.  Stock pattern:
//                            ncclAllGather, then cuBLAS GEMM.
//
// Both kernels are policies of the suite's persistent wgmma tile loop (wgmma.cuh: gemm_persistent — TMA ring,
// wgmma.mma_async into register accumulators of two consumer warpgroups, epilogue straight from the registers,
// optional CTA pairs with TMA multicast of the B tile).  Nothing in the reference is GEMM-shaped; its one collective is the ring
// allreduce (allreduce-mpi-sycl.cpp:43-67), whose fused form here is K-ring.  These two kernels are what that
// "compute step followed by a collective" idea looks like when the compute step runs on the tensor cores.
//
// Tiles are walked shard by shard starting with the neighbour (rank+1 for the reduce-scatter, the local block
// first and then rank+1, rank+2, ... for the all-gather), so at any moment the P ranks talk to P different peers
// and every NVLink carries traffic.
#include "api.h"

#include <algorithm>
#include <cstdlib>
#include <string>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "wgmma.cuh"

namespace hpcp {

namespace {

using namespace umma;

constexpr int kStages = 4;
// Shared memory left next to four 48 KiB GEMM stages and the epilogue staging: the gather thread's ring.
constexpr uint32_t kGatherSmemBytes = 14 * 1024 + 512;
constexpr int kMaxGatherBufs = 8;

// ------------------------------------------------------------------ GEMM -> reduce-scatter ----
struct RsDev {
  unsigned char* shard[kApiMaxRanks]; // peer-mapped: owner q's [M/P, N], fp32 (or bf16 when out_bf16)
  int out_bf16;
  float* c_multicast;                 // all-reduce mode: NVLS multicast mapping of fp32 [M, N]; else null
  uint32_t* done_flag[kApiMaxRanks];  // word on rank q that this rank publishes at the end (may be null)
  uint32_t done_epoch;
  uint32_t* ticket;
  uint32_t ticket_base;
  int rank, world;
  int n, k;
  int tiles_m, tiles_n;
  int shard_tiles_m;  // tiles_m / world
};

// Last CTA of the grid publishes `epoch` on every rank's flag (all threads call it).
__device__ __forceinline__ void last_cta_publish_all(uint32_t* ticket, uint32_t tickets_target,
                                                     uint32_t* const* flags, int world, uint32_t epoch) {
  const bool last = last_cta_publish(ticket, tickets_target, nullptr, 0);  // barrier + fences + ticket
  if (threadIdx.x == 0 && last)
    for (int q = 0; q < world; ++q)
      if (flags[q] != nullptr) ptx::st_release_sys(flags[q], epoch);
}

struct ReduceScatterPolicy {
  static constexpr bool kHasAuxWarp = false;
  const RsDev& g;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    shard_coords(tile, g.rank, g.world, 1, g.shard_tiles_m, g.tiles_n, m_blk, n_blk);
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    const int owner = (m0 / kBM) / g.shard_tiles_m;
    const int row0 = m0 - owner * g.shard_tiles_m * kBM + ew * kEpiRows;  // first of this warp's rows inside the shard
    const size_t elem = g.out_bf16 ? 2 : 4;
    unsigned char* base = g.shard[owner] + (static_cast<size_t>(row0) * g.n + n0) * elem;
    const size_t ld = static_cast<size_t>(g.n) * elem;
    float* stage_buf = epi_stage_buf(epi_smem, ew);
    if (g.out_bf16)
      epilogue_segments(true, d, stage_buf, lane, [&](int row, int col, int byte, const uint4& v) {
        ptx::red_add_bf16x8_sys(base + row * ld + col * 2 + byte, v);
      });
    else
      epilogue_segments(false, d, stage_buf, lane, [&](int row, int col, int byte, const uint4& v) {
        ptx::red_add_f32x4_sys(reinterpret_cast<float*>(base + row * ld + col * 4 + byte),
                               make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z),
                                           __uint_as_float(v.w)));
      });
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  __device__ __forceinline__ void finish() const {
    if (g.ticket != nullptr)
      last_cta_publish_all(g.ticket, g.ticket_base + gridDim.x, g.done_flag, g.world, g.done_epoch);
  }
};

// Reduce-scatter with the TMA unit doing the additions' issue: a consumer warp writes a [16 rows x 32 columns] fp32
// piece of its accumulator rows into a dense, 128-byte-swizzled smem tile (the 16-byte chunk c of row r goes to
// chunk c ^ (r % 8), the layout the TMA reads), and ONE cp.reduce.async.bulk.tensor.2d adds the 2 KiB tile into the
// owner's shard (UTMAREDG.2D.ADD) — 8 instructions per warp and tile instead of 1024 REDG requests through the LSU
// (wgmma.cuh: epilogue_tma_tiles).
struct RsMaps {
  CUtensorMap shard[kApiMaxRanks];  // fp32 [M/P, N] of every owner, box 16 x 32, SWIZZLE_128B
};
struct ReduceScatterTmaPolicy {
  static constexpr bool kHasAuxWarp = false;
  const RsDev& g;
  const RsMaps& maps;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    shard_coords(tile, g.rank, g.world, 1, g.shard_tiles_m, g.tiles_n, m_blk, n_blk);
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    const int owner = (m0 / kBM) / g.shard_tiles_m;
    const int y = m0 - owner * g.shard_tiles_m * kBM + ew * kEpiRows;  // first of this warp's rows inside the shard
    const CUtensorMap* map = &maps.shard[owner];
    epilogue_tma_tiles(false, d, epi_smem, ew, lane,
                       [&](const unsigned char* tile, int col) { tma_reduce_add_2d(map, n0 + col, y, tile); });
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  __device__ __forceinline__ void finish() const {
    epilogue_tma_drain();
    if (g.ticket != nullptr)
      last_cta_publish_all(g.ticket, g.ticket_base + gridDim.x, g.done_flag, g.world, g.done_epoch);
  }
};

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_reduce_scatter_tma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                                   const __grid_constant__ RsDev g, const __grid_constant__ RsMaps maps) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, ReduceScatterTmaPolicy{g, maps});
}

// All-reduce flavour: every rank adds every tile of its partial product into the multicast mapping.  The walk
// starts a 1/P-th of the tile list further for every rank (whole pairs), so the P ranks reduce into P different
// regions of C at any moment instead of queueing on the same lines of the switch.
struct AllReducePolicy {
  static constexpr bool kHasAuxWarp = false;
  const RsDev& g;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    const int num_tiles = g.tiles_m * g.tiles_n;
    const int rot = 2 * static_cast<int>(static_cast<long long>(num_tiles / 2) * g.rank / g.world);
    int t = tile + rot;
    if (t >= num_tiles) t -= num_tiles;
    tile_coords(t, g.tiles_m, g.tiles_n, m_blk, n_blk);
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    float* base = g.c_multicast + static_cast<size_t>(m0 + ew * kEpiRows) * g.n + n0;
    const size_t ld = static_cast<size_t>(g.n);
    epilogue_segments(false, d, epi_stage_buf(epi_smem, ew), lane, [&](int row, int col, int byte, const uint4& v) {
      ptx::multimem_red_add_f32x4(base + row * ld + col + byte / 4,
                                  make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z),
                                              __uint_as_float(v.w)));
    });
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  __device__ __forceinline__ void finish() const {
    if (g.ticket != nullptr)
      last_cta_publish_all(g.ticket, g.ticket_base + gridDim.x, g.done_flag, g.world, g.done_epoch);
  }
};

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_allreduce_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                          const __grid_constant__ RsDev g) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, AllReducePolicy{g});
}

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_reduce_scatter_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                               const __grid_constant__ RsDev g) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, ReduceScatterPolicy{g});
}

// ------------------------------------------------------------------ GEMM -> all-to-all ----
struct A2aDev {
  unsigned char* recv[kApiMaxRanks];  // peer-mapped: rank q's receive buffer [P, M/P, N] (fp32 or bf16)
  uint32_t* done_flag[kApiMaxRanks];
  uint32_t done_epoch;
  uint32_t* ticket;
  uint32_t ticket_base;
  int out_bf16;
  int rank, world;
  int n, k;
  int tiles_m, tiles_n;
  int shard_tiles_m;
};

struct AllToAllPolicy {
  static constexpr bool kHasAuxWarp = false;
  const A2aDev& g;
  // What the shared store epilogue needs: one destination (the owner's slot for this rank), row length, type.
  struct Out {
    void* c_local;
    void* c_peer;
    int out_bf16;
    int n;
  };
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    shard_coords(tile, g.rank, g.world, 1, g.shard_tiles_m, g.tiles_n, m_blk, n_blk);  // the neighbour's rows first
  }
  __device__ __forceinline__ void a_rows_ready(int) const {}
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    const int owner = (m0 / kBM) / g.shard_tiles_m;
    const size_t shard_rows = static_cast<size_t>(g.shard_tiles_m) * kBM;
    const size_t elem = g.out_bf16 ? 2 : 4;
    const Out out{nullptr, g.recv[owner] + static_cast<size_t>(g.rank) * shard_rows * g.n * elem, g.out_bf16, g.n};
    epilogue_store_tile(out, d, epi_stage_buf(epi_smem, ew), m0 - owner * static_cast<int>(shard_rows), n0, ew, lane);
  }
  __device__ __forceinline__ void aux_warp(int, unsigned char*) const {}
  __device__ __forceinline__ void finish() const {
    if (g.ticket != nullptr)
      last_cta_publish_all(g.ticket, g.ticket_base + gridDim.x, g.done_flag, g.world, g.done_epoch);
  }
};

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    gemm_all_to_all_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                           const __grid_constant__ A2aDev g) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, AllToAllPolicy{g});
}

// ------------------------------------------------------------------ all-gather -> GEMM ----
struct AgDev {
  unsigned char* a_full;                      // local bf16 [M, K]
  const unsigned char* a_src[kApiMaxRanks];   // peer-mapped: rank q's row block [M/P, K]
  void* c_local;                              // fp32 or bf16 [M, N]
  void* c_peer;                               // unused (kept for the shared epilogue): always null
  int out_bf16;
  int activation;                             // 0 none, 1 relu, 2 gelu (tanh form), 3 silu: applied before the store
  uint32_t* ready;                            // local [M/128] arrival counters (monotonic)
  uint32_t ready_target;                      // value a peer block's counter reaches when it is complete
  uint32_t chunk_bytes;                       // gather granularity, divides the 128-row block size
  uint32_t chunks_per_block;
  int gather_bufs;                            // depth of the gather ring (2..kMaxGatherBufs)
  uint32_t* done_flag[kApiMaxRanks];
  uint32_t done_epoch;
  uint32_t* ticket;
  uint32_t ticket_base;
  uint64_t timeout_ns;
  uint32_t* status;
  int rank, world;
  int n, k;
  int tiles_m, tiles_n;
  int shard_tiles_m;
};

struct AllGatherPolicy {
  static constexpr bool kHasAuxWarp = true;
  const AgDev& g;
  __device__ __forceinline__ void coords(int tile, int* m_blk, int* n_blk) const {
    shard_coords(tile, g.rank, g.world, 0, g.shard_tiles_m, g.tiles_n, m_blk, n_blk);  // local block first
  }
  // Producer warp, before the first A load of a tile: the rows of a peer block must have landed.  The acquire
  // pairs with the gather warps' release increments; the proxy fence orders it before this thread's TMA loads.
  __device__ __forceinline__ void a_rows_ready(int m_blk) const {
    if (m_blk / g.shard_tiles_m != g.rank) {
      if ((threadIdx.x & 31) == 0) {
        (void)wait_epoch(&g.ready[m_blk], g.ready_target, g.timeout_ns, g.status);
        asm volatile("fence.proxy.async;" ::: "memory");
      }
      __syncwarp();
    }
  }
  __device__ __forceinline__ void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew,
                                           int lane) const {
    float* stage_buf = epi_stage_buf(epi_smem, ew);
    if (g.activation == 0) {
      epilogue_store_tile(g, d, stage_buf, m0, n0, ew, lane);
      return;
    }
    // Fused activation (the layer's nonlinearity never costs a pass over C in HBM).
    const size_t elem = g.out_bf16 ? 2 : 4;
    unsigned char* base =
        static_cast<unsigned char*>(g.c_local) + (static_cast<size_t>(m0 + ew * kEpiRows) * g.n + n0) * elem;
    const size_t ld = static_cast<size_t>(g.n) * elem;
    auto store = [&](int row, int col, int byte, const uint4& v) {
      *reinterpret_cast<uint4*>(base + row * ld + col * elem + byte) = v;
    };
    if (g.activation == 1)
      epilogue_segments(g.out_bf16 != 0, d, stage_buf, lane, store, [](float x) { return fmaxf(x, 0.0f); });
    else if (g.activation == 2)
      epilogue_segments(g.out_bf16 != 0, d, stage_buf, lane, store, [](float x) {
        float t;  // gelu, tanh form: 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
        asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.7978845608f * (x + 0.044715f * x * x * x)));
        return 0.5f * x * (1.0f + t);
      });
    else
      epilogue_segments(g.out_bf16 != 0, d, stage_buf, lane, store,
                        [](float x) { return __fdividef(x, 1.0f + __expf(-x)); });  // silu
  }
  // Gather engine: one thread per CTA streams its share of the peers' row blocks, peer (rank+1) first — the
  // order in which the tile loop needs them.  Piece c of the (P-1) * M/P * K * 2 remote bytes belongs to CTA
  // c % gridDim.x, so the pieces of a block are spread over all SMs and the block completes as early as possible.
  __device__ __forceinline__ void aux_warp(int lane, unsigned char* aux_smem) const {
    if (lane == 0 && g.world > 1) gather(aux_smem);
    __syncwarp();
  }
  __device__ __forceinline__ void gather(unsigned char* aux_smem) const {
    const int bufs = g.gather_bufs;
    uint64_t* full = reinterpret_cast<uint64_t*>(aux_smem + static_cast<size_t>(bufs) * g.chunk_bytes);
    for (int s = 0; s < bufs; ++s) ptx::mbar_init(&full[s], 1);
    ptx::fence_mbar_init();
    const size_t block_bytes = static_cast<size_t>(kBM) * g.k * 2;
    const size_t total = static_cast<size_t>(g.world - 1) * g.shard_tiles_m * g.chunks_per_block;
    const size_t n = total > blockIdx.x ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto piece = [&](size_t j) {  // my j-th piece (tile_order.h: peer rank+1 first, pieces dealt round-robin)
      return gather_piece(static_cast<size_t>(blockIdx.x) + j * gridDim.x, g.rank, g.world, g.shard_tiles_m,
                          g.chunks_per_block, g.chunk_bytes, block_bytes);
    };
    auto issue_load = [&](size_t j) {
      const int st = static_cast<int>(j % bufs);
      ptx::mbar_arrive_expect_tx(&full[st], g.chunk_bytes);
      const GatherPiece p = piece(j);
      ptx::bulk_g2s(aux_smem + static_cast<size_t>(st) * g.chunk_bytes, g.a_src[p.peer] + p.src_off, g.chunk_bytes,
                    &full[st]);
    };
    // Stores are retired in order: once store j-1 is complete its piece is counted and its buffer is reused.
    auto retire = [&](size_t j) {
      asm volatile("fence.proxy.async;" ::: "memory");
      ptx::red_release_gpu_add(g.ready + piece(j).m_blk, 1u);
    };
    const size_t lookahead = static_cast<size_t>(bufs - 1);
    for (size_t j = 0; j < lookahead && j < n; ++j) issue_load(j);
    for (size_t j = 0; j < n; ++j) {
      const int st = static_cast<int>(j % bufs);
      ptx::mbar_wait(&full[st], static_cast<uint32_t>((j / bufs) & 1));
      ptx::bulk_s2g(g.a_full + piece(j).dst_off, aux_smem + static_cast<size_t>(st) * g.chunk_bytes, g.chunk_bytes);
      ptx::bulk_commit();
      if (j > 0) {
        ptx::bulk_wait<1>();  // every store but the newest is complete (written, not just read)
        retire(j - 1);
      }
      if (j + lookahead < n) issue_load(j + lookahead);  // into the buffer store j-1 has just left
    }
    if (n > 0) {
      ptx::bulk_wait<0>();
      retire(n - 1);
    }
  }
  // The arrival epoch tells every peer that this rank no longer reads its row block.
  __device__ __forceinline__ void finish() const {
    if (g.ticket != nullptr)
      last_cta_publish_all(g.ticket, g.ticket_base + gridDim.x, g.done_flag, g.world, g.done_epoch);
  }
};

template <int kCluster>
__global__ void __launch_bounds__(kThreads, 1)
    allgather_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                          const __grid_constant__ AgDev g) {
  gemm_persistent<kCluster, kStages>(map_a, map_b, g.tiles_m, g.tiles_n, g.k, AllGatherPolicy{g});
}

// ------------------------------------------------------------------ wait for P flags ----
__global__ void __launch_bounds__(32) wait_flags_kernel(const uint32_t* flags, int count, uint32_t epoch,
                                                        uint64_t timeout_ns, uint32_t* status) {
  if (static_cast<int>(threadIdx.x) < count) (void)wait_epoch(flags + threadIdx.x, epoch, timeout_ns, status);
}

// Shapes both kernels accept: whole 128x256x64 tiles, whole tiles per shard, and (for CTA pairs) an even number
// of tile rows per raster group inside a shard.
struct Shape {
  int tiles_m, tiles_n, shard_tiles_m;
  bool pairable;
};
Shape check_shape(const char* who, int m, int n, int k, int world) {
  const std::string w(who);
  HPCP_REQUIRE(world >= 1 && world <= kApiMaxRanks, w + ": world must be in [1,16]");
  HPCP_REQUIRE(m > 0 && n > 0 && k > 0 && m % kBM == 0 && n % kBN == 0 && k % kBK == 0,
               w + ": M, N, K must be multiples of 128, 256, 64");
  HPCP_REQUIRE((m / kBM) % world == 0, w + ": M must be a multiple of 128 * world (whole tiles per shard)");
  Shape s;
  s.tiles_m = m / kBM;
  s.tiles_n = n / kBN;
  s.shard_tiles_m = s.tiles_m / world;
  s.pairable = s.shard_tiles_m % 2 == 0 && (s.shard_tiles_m % kGroupM) % 2 == 0;
  return s;
}

template <class Kernel, class... Args>
void launch_pairs(Kernel kernel, int grid, size_t smem, cudaStream_t stream, const Args&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(grid));
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
  HPCP_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
}

// One launch of a tile-loop kernel family: `single` on plain CTAs (B box = the whole 256-row tile), or `pair` on
// clusters of two (each CTA fetches half of the B tile: box = 128 rows).  Returns the number of CTAs launched.
template <class Single, class Pair, class... Rest>
int launch_tile_loop(Single single, Pair pair, bool pairs, int grid, size_t smem_single, size_t smem_pair,
                     cudaStream_t stream, const CUtensorMap& map_a, const void* b, int n, int k, const Rest&... rest) {
  if (!pairs || grid < 2) {
    const CUtensorMap map_b = make_kmajor_map(b, n, k, kBN);
    HPCP_ENABLE_SMEM(single, smem_single);
    single<<<grid, kThreads, smem_single, stream>>>(map_a, map_b, rest...);
    HPCP_CUDA(cudaGetLastError());
    return grid;
  }
  grid &= ~1;  // whole pairs
  const CUtensorMap map_b = make_kmajor_map(b, n, k, kBN / 2);
  HPCP_ENABLE_SMEM(pair, smem_pair);
  launch_pairs(pair, grid, smem_pair, stream, map_a, map_b, rest...);
  return grid;
}

}  // namespace

void launch_wait_flags(const uint32_t* flags, int count, uint32_t epoch, uint64_t timeout_ns, uint32_t* status,
                       cudaStream_t stream) {
  HPCP_REQUIRE(count >= 0 && count <= 32, "wait_flags: at most 32 consecutive words");
  if (count == 0) return;
  wait_flags_kernel<<<1, 32, 0, stream>>>(flags, count, epoch, timeout_ns, status);
  HPCP_CUDA(cudaGetLastError());
}

int launch_gemm_reduce_scatter(const GemmRsArgs& args, int ctas, int device, cudaStream_t stream, int cluster) {
  const Shape s = check_shape("gemm_reduce_scatter", args.m, args.n, args.k, args.world);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "gemm_reduce_scatter: bad rank");
  HPCP_REQUIRE(cluster >= 0 && cluster <= 2, "gemm_reduce_scatter: cluster must be 0 (auto), 1 or 2");
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(args.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(args.b) & 15) == 0,
               "gemm_reduce_scatter: operands must be 16-byte aligned");
  RsDev g{};
  const bool all_reduce = args.c_multicast != nullptr;
  HPCP_REQUIRE(!all_reduce || (reinterpret_cast<uintptr_t>(args.c_multicast) & 15) == 0,
               "gemm_reduce_scatter: the multicast mapping must be 16-byte aligned");
  g.c_multicast = args.c_multicast;
  HPCP_REQUIRE(!all_reduce || !args.out_bf16, "gemm_reduce_scatter: the all-reduce flavour accumulates in fp32");
  g.out_bf16 = args.out_bf16 ? 1 : 0;
  for (int q = 0; q < args.world; ++q) {
    HPCP_REQUIRE(all_reduce || (args.shard[q] != nullptr && (reinterpret_cast<uintptr_t>(args.shard[q]) & 15) == 0),
                 "gemm_reduce_scatter: every rank's shard pointer is needed (16-byte aligned)");
    g.shard[q] = static_cast<unsigned char*>(args.shard[q]);
    g.done_flag[q] = args.done_flag[q];
    HPCP_REQUIRE(args.done_flag[q] == nullptr || args.ticket != nullptr,
                 "gemm_reduce_scatter: a signal needs a ticket counter");
  }
  g.done_epoch = args.done_epoch;
  g.ticket = args.ticket;
  g.ticket_base = args.ticket_base;
  g.rank = args.rank;
  g.world = args.world;
  g.n = args.n;
  g.k = args.k;
  g.tiles_m = s.tiles_m;
  g.tiles_n = s.tiles_n;
  g.shard_tiles_m = s.shard_tiles_m;
  // Pairs of the all-reduce flavour walk the whole C in the grouped order: the usual whole-matrix condition.
  const bool pairable = all_reduce ? (s.tiles_m % 2 == 0 && (s.tiles_m % kGroupM) % 2 == 0) : s.pairable;
  HPCP_REQUIRE(cluster != 2 || pairable, "gemm_reduce_scatter: cluster=2 needs an even number of tile rows per group");
  const bool pairs = cluster != 1 && pairable;
  const CUtensorMap map_a = make_kmajor_map(args.a, args.m, args.k, kBM);
  const int tiles = s.tiles_m * s.tiles_n;
  int grid = std::min(tiles, ctas > 0 ? ctas : device_sm_count(device));
  constexpr size_t smem = gemm_smem_bytes<kStages>(0);
  if (args.tma_epilogue) {  // additions issued by the TMA unit (UTMAREDG) instead of REDG requests from the LSU
    HPCP_REQUIRE(!all_reduce && !args.out_bf16, "gemm_reduce_scatter: the TMA epilogue exists for fp32 shards");
    RsMaps maps{};
    for (int q = 0; q < args.world; ++q) maps.shard[q] = make_c_tile_map(args.shard[q], args.m / args.world, args.n, false);
    constexpr size_t smem_t = gemm_smem_bytes<kStages>(kTmaEpiSmemBytes - kEpiWarps * kEpiWarpBytes);
    static_assert(smem_t + 1024 <= 227 * 1024, "GEMM stages + two reduce tiles per epilogue warp must fit in 227 KiB");
    return launch_tile_loop(gemm_reduce_scatter_tma_kernel<1>, gemm_reduce_scatter_tma_kernel<2>, pairs, grid, smem_t,
                            smem_t, stream, map_a, args.b, args.n, args.k, g, maps);
  }
  if (all_reduce)
    return launch_tile_loop(gemm_allreduce_kernel<1>, gemm_allreduce_kernel<2>, pairs, grid, smem, smem, stream, map_a,
                            args.b, args.n, args.k, g);
  return launch_tile_loop(gemm_reduce_scatter_kernel<1>, gemm_reduce_scatter_kernel<2>, pairs, grid, smem, smem, stream,
                          map_a, args.b, args.n, args.k, g);
}

int launch_gemm_all_to_all(const GemmA2aArgs& args, int ctas, int device, cudaStream_t stream, int cluster) {
  const Shape s = check_shape("gemm_all_to_all", args.m, args.n, args.k, args.world);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "gemm_all_to_all: bad rank");
  HPCP_REQUIRE(cluster >= 0 && cluster <= 2, "gemm_all_to_all: cluster must be 0 (auto), 1 or 2");
  HPCP_REQUIRE(cluster != 2 || s.pairable, "gemm_all_to_all: cluster=2 needs an even number of tile rows per shard");
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(args.a) & 15) == 0 && (reinterpret_cast<uintptr_t>(args.b) & 15) == 0,
               "gemm_all_to_all: operands must be 16-byte aligned");
  A2aDev g{};
  for (int q = 0; q < args.world; ++q) {
    HPCP_REQUIRE(args.recv[q] != nullptr && (reinterpret_cast<uintptr_t>(args.recv[q]) & 15) == 0,
                 "gemm_all_to_all: every rank's receive buffer is needed (16-byte aligned)");
    g.recv[q] = static_cast<unsigned char*>(args.recv[q]);
    g.done_flag[q] = args.done_flag[q];
    HPCP_REQUIRE(args.done_flag[q] == nullptr || args.ticket != nullptr, "gemm_all_to_all: a signal needs a ticket counter");
  }
  g.done_epoch = args.done_epoch;
  g.ticket = args.ticket;
  g.ticket_base = args.ticket_base;
  g.out_bf16 = args.out_bf16 ? 1 : 0;
  g.rank = args.rank;
  g.world = args.world;
  g.n = args.n;
  g.k = args.k;
  g.tiles_m = s.tiles_m;
  g.tiles_n = s.tiles_n;
  g.shard_tiles_m = s.shard_tiles_m;
  const bool pairs = cluster != 1 && s.pairable;
  const CUtensorMap map_a = make_kmajor_map(args.a, args.m, args.k, kBM);
  int grid = std::min(s.tiles_m * s.tiles_n, ctas > 0 ? ctas : device_sm_count(device));
  constexpr size_t smem = gemm_smem_bytes<kStages>(0);
  return launch_tile_loop(gemm_all_to_all_kernel<1>, gemm_all_to_all_kernel<2>, pairs, grid, smem, smem, stream, map_a,
                          args.b, args.n, args.k, g);
}

uint32_t allgather_gemm_chunks_per_block(int k, int chunk_bytes) {
  const int chunk = chunk_bytes > 0 ? chunk_bytes : 4096;
  return static_cast<uint32_t>(static_cast<size_t>(kBM) * k * 2 / chunk);
}

int launch_allgather_gemm(const AgGemmArgs& args, int ctas, int device, cudaStream_t stream, int cluster) {
  const Shape s = check_shape("allgather_gemm", args.m, args.n, args.k, args.world);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "allgather_gemm: bad rank");
  HPCP_REQUIRE(cluster >= 0 && cluster <= 2, "allgather_gemm: cluster must be 0 (auto), 1 or 2");
  HPCP_REQUIRE(cluster != 2 || s.pairable, "allgather_gemm: cluster=2 needs an even number of tile rows per shard");
  HPCP_REQUIRE(args.a_full != nullptr && args.b != nullptr && args.c != nullptr, "allgather_gemm: null operand");
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(args.a_full) & 127) == 0 && (reinterpret_cast<uintptr_t>(args.b) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(args.c) & 15) == 0,
               "allgather_gemm: a_full must be 128-byte aligned, b and c 16-byte aligned");
  const int chunk = args.chunk_bytes > 0 ? args.chunk_bytes : 4096;
  const size_t block_bytes = static_cast<size_t>(kBM) * args.k * 2;
  HPCP_REQUIRE(chunk % 16 == 0 && chunk >= 512 && chunk <= 4096 && block_bytes % chunk == 0,
               "allgather_gemm: chunk_bytes must be a multiple of 16 in [512, 4096] that divides 256*K");
  HPCP_REQUIRE(args.world == 1 || args.ready != nullptr, "allgather_gemm: the arrival counters are needed");
  AgDev g{};
  for (int q = 0; q < args.world; ++q) {
    HPCP_REQUIRE(q == args.rank || (args.a_src[q] != nullptr && (reinterpret_cast<uintptr_t>(args.a_src[q]) & 15) == 0),
                 "allgather_gemm: every peer's row block pointer is needed (16-byte aligned)");
    g.a_src[q] = static_cast<const unsigned char*>(args.a_src[q]);
    g.done_flag[q] = args.done_flag[q];
    HPCP_REQUIRE(args.done_flag[q] == nullptr || args.ticket != nullptr, "allgather_gemm: a signal needs a ticket counter");
  }
  g.a_full = static_cast<unsigned char*>(args.a_full);
  g.c_local = args.c;
  g.c_peer = nullptr;
  g.out_bf16 = args.out_bf16 ? 1 : 0;
  HPCP_REQUIRE(args.activation >= 0 && args.activation <= 3, "allgather_gemm: activation must be 0..3");
  g.activation = args.activation;
  g.ready = args.ready;
  g.chunk_bytes = static_cast<uint32_t>(chunk);
  g.chunks_per_block = static_cast<uint32_t>(block_bytes / chunk);
  g.gather_bufs = std::min<int>(kMaxGatherBufs, static_cast<int>((kGatherSmemBytes - 64) / chunk));
  g.ready_target = args.ready_base + g.chunks_per_block;
  g.done_epoch = args.done_epoch;
  g.ticket = args.ticket;
  g.ticket_base = args.ticket_base;
  g.timeout_ns = args.timeout_ns;
  g.status = args.status;
  g.rank = args.rank;
  g.world = args.world;
  g.n = args.n;
  g.k = args.k;
  g.tiles_m = s.tiles_m;
  g.tiles_n = s.tiles_n;
  g.shard_tiles_m = s.shard_tiles_m;
  const bool pairs = cluster != 1 && s.pairable;
  const CUtensorMap map_a = make_kmajor_map(args.a_full, args.m, args.k, kBM);
  const int tiles = s.tiles_m * s.tiles_n;
  // Every CTA carries a share of the gather, so the whole grid must be resident: never more CTAs than SMs.
  int grid = std::min(tiles, std::min(ctas > 0 ? ctas : device_sm_count(device), device_sm_count(device)));
  constexpr size_t smem = gemm_smem_bytes<kStages>(kGatherSmemBytes);
  static_assert(smem + 1024 <= 227 * 1024,  // + the static barriers, padded to the 1 KiB alignment of the ring
                "GEMM stages + epilogue staging + gather ring must fit in 227 KiB");
  if (pairs && grid >= 2) {
    // Not every SM can host half of a CTA pair (a GPC may have an SM left over): never more pairs than fit at once.
    HPCP_ENABLE_SMEM(allgather_gemm_kernel<2>, smem);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(grid & ~1));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    HPCP_CUDA(cudaOccupancyMaxActiveClusters(&clusters, allgather_gemm_kernel<2>, &cfg));
    HPCP_REQUIRE(clusters >= 1, "allgather_gemm: no CTA pair fits on this device");
    grid = std::min(grid, 2 * clusters);
  }
  return launch_tile_loop(allgather_gemm_kernel<1>, allgather_gemm_kernel<2>, pairs, grid, smem, smem, stream, map_a,
                          args.b, args.n, args.k, g);
}

}  // namespace hpcp
