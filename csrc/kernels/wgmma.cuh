// Warpgroup-MMA (wgmma) building blocks shared by the tensor-core kernels of the suite (gemm_put.cu, gemm_collective.cu,
// tc_payload.cu): tile geometry, the shared-memory matrix descriptor, TMA tensor loads / stores / reductions,
// wgmma.mma_async wrappers, the epilogue walks over the register accumulator, the persistent tile loop and the
// host-side tensor-map encoder.  Everything device-side is __forceinline__.
#pragma once

#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>

#include <cstdio>
#include <mutex>
#include <string>

#include "../common/cuda_check.h"
#include "../common/ptx.cuh"
#include "tile_order.h"

namespace hpcp {
namespace umma {

constexpr int kBM = 128, kBN = 256, kBK = 64, kMmaK = 16;
// Warpgroup 0: TMA producer (warp 0) and the policy's aux warp (warp 3).  Warpgroups 1 and 2: consumers, each owns
// 64 rows of the 128x256 tile as a wgmma m64n256 fp32 accumulator in registers (128 per thread) and stores it itself.
constexpr int kThreads = 384;
constexpr int kConsumers = 2;
constexpr int kEpiWarps = 4 * kConsumers;              // consumer warp ew owns tile rows [16 ew, 16 ew + 16)
constexpr int kEpiRows = 16;
constexpr int kAccRegs = kBN / 2;                      // fp32 accumulator registers per consumer thread
constexpr uint32_t kABytes = kBM * kBK * 2;            // 16 KiB
constexpr uint32_t kBBytes = kBN * kBK * 2;            // 32 KiB
constexpr int kStageRowWords = 36;                     // 32 payload floats + 4 pad (keeps float4 alignment)
constexpr uint32_t kEpiWarpBytes = kEpiRows * kStageRowWords * 4;  // 2304 B per consumer warp

// ---- shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format" of wgmma) ----
// K-major, SWIZZLE_128B: 8-row x 128-byte atoms stacked every 1024 bytes (stride byte offset); the leading byte
// offset is unused for swizzled K-major layouts (encoded 1); base offset 0 (every tile is 1024-byte aligned);
// layout type 1 = SWIZZLE_128B.  Advancing K by 16 bf16 inside the atom adds 32 bytes to the start address.
__host__ __device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);  // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                      // LBO            [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // SBO            [32,46): 8 rows x 128 B
  d |= static_cast<uint64_t>(1) << 62;                      // SWIZZLE_128B   [62,64)
  return d;
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int x, int y,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3}], [%4];" ::"r"(ptx::smem_u32(smem_dst)),
      "l"(map), "r"(x), "r"(y), "r"(ptx::smem_u32(bar))
      : "memory");
}
// Multicast variant: the box lands at the same smem offset in every CTA of `cta_mask`, and each of
// those CTAs' mbarrier (same offset) receives the complete_tx.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, int x, int y,
                                                      uint64_t* bar, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%2, %3}], [%4], %5;" ::"r"(ptx::smem_u32(smem_dst)),
      "l"(map), "r"(x), "r"(y), "r"(ptx::smem_u32(bar)), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_cta_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Arrive on the barrier at the same offset in CTA `cta` of the cluster (the own CTA included).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(ptx::smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// ---- wgmma ----
// D[64 x 256] (fp32, registers) (+)= A[64 x 16] . B[256 x 16]^T, both operands bf16 K-major in shared memory.
// Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4j + h] is row 16 w + l / 4 + 8 (h / 2),
// column 8 j + 2 (l % 4) + h % 2.
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[kAccRegs], uint64_t desc_a, uint64_t desc_b,
                                                      uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Pins the accumulator registers at this point of the instruction stream, so that no register work on them (the
// epilogue's conversions, a fused activation) can be scheduled across an MMA issue or a wgmma.wait_group
// (CUTLASS: warpgroup_fence_operand).
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[kAccRegs]) {
#pragma unroll
  for (int i = 0; i < kAccRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// The four K=16 steps of one 64-deep k-block of the warpgroup's 64 rows.
__device__ __forceinline__ void wgmma_kblock(float (&d)[kAccRegs], uint32_t sa, uint32_t sb, bool accumulate) {
  const uint64_t desc_a = make_smem_desc(sa);
  const uint64_t desc_b = make_smem_desc(sb);
#pragma unroll
  for (int kk = 0; kk < kBK / kMmaK; ++kk) {
    const uint64_t adv = static_cast<uint64_t>((kk * kMmaK * 2) >> 4);
    wgmma_m64n256k16_bf16(d, desc_a + adv, desc_b + adv, (accumulate || kk != 0) ? 1u : 0u);
  }
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

// Epilogue walk of one consumer warp's 16 accumulator rows: registers -> padded smem staging -> 16-byte pieces of
// full 128-byte row segments.  One round moves a 128-byte segment per row: 32 fp32 columns, or 64 bf16 columns
// (converted before staging), so whatever emit() does with a piece (store, peer store, reduction) always happens in
// full 128-byte segments: 8 consecutive lanes = one segment, 4 rows per instruction.  emit(row, col, byte, v): 16
// bytes `v` of accumulator row `row` (0..15 inside this warp's rows) that start `byte` bytes into the round's
// segment, whose first column is `col`.
// pre(x): applied to every fp32 accumulator value before it is converted / staged (a fused activation).
struct EpilogueIdentity {
  __device__ __forceinline__ float operator()(float x) const { return x; }
};
template <class Emit, class Pre = EpilogueIdentity>
__device__ __forceinline__ void epilogue_segments(bool out_bf16, const float (&d)[kAccRegs], float* stage_buf,
                                                  int lane, Emit emit, Pre pre = Pre{}) {
  unsigned char* stage = reinterpret_cast<unsigned char*>(stage_buf);
  const int r0 = lane >> 2;            // fragment rows r0 and r0 + 8
  const int cq = 2 * (lane & 3);       // fragment column inside each group of 8
  auto round = [&](int col, auto stage_round) {
    stage_round(col);
    __syncwarp();
#pragma unroll
    for (int it = 0; it < kEpiRows / 4; ++it) {
      const int row = it * 4 + (lane >> 3);
      const int c16 = lane & 7;
      const uint4 v = *reinterpret_cast<const uint4*>(stage + row * (kStageRowWords * 4) + c16 * 16);
      emit(row, col, c16 * 16, v);
    }
    __syncwarp();
  };
  if (out_bf16) {
#pragma unroll
    for (int col = 0; col < kBN; col += 64)
      round(col, [&](int c0) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = c0 / 8 + jj;
          const int byte = (8 * jj + cq) * 2;
          *reinterpret_cast<uint32_t*>(stage + r0 * (kStageRowWords * 4) + byte) =
              pack_bf16x2(pre(d[4 * j]), pre(d[4 * j + 1]));
          *reinterpret_cast<uint32_t*>(stage + (r0 + 8) * (kStageRowWords * 4) + byte) =
              pack_bf16x2(pre(d[4 * j + 2]), pre(d[4 * j + 3]));
        }
      });
  } else {
#pragma unroll
    for (int col = 0; col < kBN; col += 32)
      round(col, [&](int c0) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = c0 / 8 + jj;
          const int byte = (8 * jj + cq) * 4;
          *reinterpret_cast<float2*>(stage + r0 * (kStageRowWords * 4) + byte) =
              make_float2(pre(d[4 * j]), pre(d[4 * j + 1]));
          *reinterpret_cast<float2*>(stage + (r0 + 8) * (kStageRowWords * 4) + byte) =
              make_float2(pre(d[4 * j + 2]), pre(d[4 * j + 3]));
        }
      });
  }
}

// The plain epilogue: the walk above storing to c_local and/or c_peer (streaming stores for the peer copy).
// G: any struct with c_local, c_peer (either may be null), out_bf16 and n (the row length of C).
template <class G>
__device__ __forceinline__ void epilogue_store_tile(const G& g, const float (&d)[kAccRegs], float* stage_buf, int m0,
                                                    int n0, int ew, int lane) {
  const size_t elem = g.out_bf16 ? 2 : 4;
  epilogue_segments(g.out_bf16 != 0, d, stage_buf, lane, [&](int row, int col, int byte, const uint4& v) {
    const size_t off = (static_cast<size_t>(m0 + ew * kEpiRows + row) * g.n + n0 + col) * elem + byte;
    if (g.c_peer != nullptr) ptx::st_stream_v4(reinterpret_cast<uint4*>(static_cast<unsigned char*>(g.c_peer) + off), v);
    if (g.c_local != nullptr) *reinterpret_cast<uint4*>(static_cast<unsigned char*>(g.c_local) + off) = v;
  });
}

// smem [16 x 128 B] tile (SWIZZLE_128B layout, 1024-byte aligned) added into a 2-D fp32 tensor at element (x, y) by
// the TMA unit: one instruction per 2 KiB instead of 128 REDG requests from the LSU.
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, int x, int y, const void* smem_src) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(map),
               "r"(x), "r"(y), "r"(ptx::smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int x, int y, const void* smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(map), "r"(x),
               "r"(y), "r"(ptx::smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Epilogue walk for the TMA unit: the warp's 16 accumulator rows leave in [16 rows x 128 bytes] pieces (32 fp32 or
// 64 bf16 columns) staged in dense, 128-byte-swizzled shared memory — the 16-byte chunk c of row r goes to chunk
// c ^ (r % 8), the layout a SWIZZLE_128B tensor map expects — and lane 0 calls issue(tile, col) (one or more
// cp.async.bulk.tensor / cp.reduce.async.bulk.tensor instructions on a tensor map with a 16-row x 128-byte box), which
// this function commits as one bulk group.  Two 2 KiB tiles per warp, carved out of the (1024-byte aligned)
// epilogue area: the TMA reads one while the warp fills the other.
// The caller's finish() must wait for the groups (epilogue_tma_drain) before it signals anything.
constexpr uint32_t kTmaTileBytes = kEpiRows * 128;
constexpr uint32_t kTmaEpiSmemBytes = kEpiWarps * 2 * kTmaTileBytes;  // 32 KiB instead of the 18 KiB staging
template <class Issue>
__device__ __forceinline__ void epilogue_tma_tiles(bool out_bf16, const float (&d)[kAccRegs], unsigned char* epi_smem,
                                                   int ew, int lane, Issue issue) {
  unsigned char* tiles = epi_smem + static_cast<size_t>(ew) * 2 * kTmaTileBytes;
  const int r0 = lane >> 2;
  const int cq = 2 * (lane & 3);
  // byte b of row r of a swizzled tile
  auto at = [&](unsigned char* tile, int r, int b) { return tile + r * 128 + (((b >> 4) ^ (r & 7)) << 4) + (b & 15); };
  auto round = [&](int col, int parity, auto fill) {
    unsigned char* tile = tiles + parity * kTmaTileBytes;
    // The group issued two rounds ago used this tile: it must have finished READING it (groups are per thread, lane
    // 0 issued them all; at most the newest one — the other tile — may still be pending).
    if (lane == 0) ptx::bulk_wait_read<1>();
    __syncwarp();
    fill(tile, col);
    fence_proxy_async_smem();  // my generic-proxy writes before the async-proxy read of the tile
    __syncwarp();
    if (lane == 0) {
      issue(tile, col);
      ptx::bulk_commit();
    }
  };
  // The accumulator is indexed with constants only (fully unrolled loops), so it stays in registers.
  if (out_bf16) {
#pragma unroll
    for (int col = 0; col < kBN; col += 64)
      round(col, (col / 64) & 1, [&](unsigned char* tile, int c0) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = c0 / 8 + jj;
          const int b = (8 * jj + cq) * 2;
          *reinterpret_cast<uint32_t*>(at(tile, r0, b)) = pack_bf16x2(d[4 * j], d[4 * j + 1]);
          *reinterpret_cast<uint32_t*>(at(tile, r0 + 8, b)) = pack_bf16x2(d[4 * j + 2], d[4 * j + 3]);
        }
      });
  } else {
#pragma unroll
    for (int col = 0; col < kBN; col += 32)
      round(col, (col / 32) & 1, [&](unsigned char* tile, int c0) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = c0 / 8 + jj;
          const int b = (8 * jj + cq) * 4;
          *reinterpret_cast<float2*>(at(tile, r0, b)) = make_float2(d[4 * j], d[4 * j + 1]);
          *reinterpret_cast<float2*>(at(tile, r0 + 8, b)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
        }
      });
  }
}
// finish() part of the TMA epilogues: every bulk group of this CTA must be PERFORMED before anything is signalled
// (and must have stopped reading shared memory before the CTA retires).
__device__ __forceinline__ void epilogue_tma_drain() {
  if (threadIdx.x >= 128 && (threadIdx.x & 31) == 0) {
    ptx::bulk_wait<0>();
    asm volatile("fence.proxy.async;" ::: "memory");
  }
}

// ---------------------------------------------------------------- persistent GEMM main loop ----
// The warp-specialised persistent tile loop every GEMM kernel of the suite runs (384 threads, one CTA per SM):
//   warp 0        TMA producer : A[128x64] + B[256x64] per stage, kStagesT-deep smem ring, full/empty mbarriers
//   warp 3        policy.aux_warp(): idle for a plain GEMM, the gather engine of all-gather -> GEMM
//   warpgroups 1,2 consumers   : wgmma m64n256k16 over their 64 rows of A and the whole B stage, fp32 accumulator in
//                                registers; a stage is released once the wgmma reading it has completed (one k-block
//                                of MMAs stays in flight), then policy.epilogue() stores the tile while the producer
//                                already fills the ring for the next one.
// kCluster == 2: clusters of two CTAs working on vertically adjacent tiles (same n_blk).  Both need the same B
// tile, so each CTA fetches half of it (128 rows) and TMA-multicasts it into both CTAs' shared memory:
// L2->SM operand traffic drops from 48 to 32 KiB per CTA per k-block.  A stage may only be refilled when the
// consumers of BOTH CTAs have finished with it: the empty barriers count 2 x kConsumers arrivals, and every consumer
// warpgroup arrives in both CTAs.
//
// What differs between the kernels is the Policy:
//   void coords(int tile, int* m_blk, int* n_blk) const    tile index -> tile coordinates (rasterisation)
//   void a_rows_ready(int m_blk) const                      producer warp, before the first A load of a tile
//   void epilogue(const float (&d)[kAccRegs], unsigned char* epi_smem, int m0, int n0, int ew, int lane) const
//                                                           consumer warp ew: its rows [m0 + 16 ew, +16) of the tile
//   void aux_warp(int lane, unsigned char* aux_smem) const  warp 3, runs concurrently with the tile loop
//   void finish() const                                     all threads, after the loop
//   static constexpr bool kHasAuxWarp                       false: warp 3 idles (the branch is compiled out)
// epi_smem is the epilogue area (kEpiWarps * kEpiWarpBytes, or more if the launcher asked for it); aux_smem points
// behind the epilogue staging buffers, its size is whatever the launcher added to gemm_smem_bytes<kStagesT>(aux_bytes).
template <int kStagesT>
constexpr size_t gemm_smem_bytes(uint32_t aux_bytes) {
  return static_cast<size_t>(kStagesT) * (kABytes + kBBytes) + kEpiWarps * kEpiWarpBytes + aux_bytes + 1024;
}
// Staging buffer of consumer warp ew inside the epilogue area.
__device__ __forceinline__ float* epi_stage_buf(unsigned char* epi_smem, int ew) {
  return reinterpret_cast<float*>(epi_smem + static_cast<size_t>(ew) * kEpiWarpBytes);
}

template <int kCluster, int kStagesT, class Policy>
__device__ __forceinline__ void gemm_persistent(const CUtensorMap& map_a, const CUtensorMap& map_b, int tiles_m,
                                                int tiles_n, int k, const Policy& policy) {
  constexpr uint32_t kStageBytesT = kABytes + kBBytes;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStagesT];
  __shared__ __align__(8) uint64_t empty_bar[kStagesT];

  unsigned char* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* epi_smem = smem + static_cast<size_t>(kStagesT) * kStageBytesT;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = k / kBK;
  const int crank = kCluster > 1 ? static_cast<int>(cluster_cta_rank()) : 0;
  // Work items are tile pairs in cluster mode: pair p -> tiles 2p, 2p+1 (consecutive tiles of the
  // grouped rasterisation share n_blk when the group height is even).
  const int first_item = static_cast<int>(blockIdx.x) / kCluster;
  const int item_stride = static_cast<int>(gridDim.x) / kCluster;
  const int num_items = num_tiles / kCluster;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
    for (int s = 0; s < kStagesT; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kConsumers * kCluster);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (kCluster > 1) cluster_sync_all();  // the peer's barriers exist before anything remote touches them

  if (warp == 0) {
    // ===================== TMA producer =====================
    // The whole warp walks the loop (convergent barriers at kernel end); lane 0 issues the TMA.
    int stage = 0;
    uint32_t phase = 0;
    for (int item = first_item; item < num_items; item += item_stride) {
      const int tile = item * kCluster + crank;
      int m_blk, n_blk;
      policy.coords(tile, &m_blk, &n_blk);
      const int m0 = m_blk * kBM;
      const int n0 = n_blk * kBN;
      policy.a_rows_ready(m_blk);
      for (int kb = 0; kb < num_kb; ++kb) {
        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);  // slot released by the consumers (of both CTAs)
        if (lane == 0) {
          unsigned char* sa = smem + static_cast<size_t>(stage) * kStageBytesT;
          ptx::mbar_arrive_expect_tx(&full_bar[stage], kStageBytesT);
          tma_load_2d(sa, &map_a, kb * kBK, m0, &full_bar[stage]);
          if (kCluster > 1)  // my half of the shared B tile, delivered to both CTAs of the pair
            tma_load_2d_multicast(sa + kABytes + crank * (kBBytes / 2), &map_b, kb * kBK,
                                  n0 + crank * (kBN / 2), &full_bar[stage], static_cast<uint16_t>(0x3));
          else
            tma_load_2d(sa + kABytes, &map_b, kb * kBK, n0, &full_bar[stage]);
        }
        __syncwarp();
        if (++stage == kStagesT) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (Policy::kHasAuxWarp && warp == 3) {
    policy.aux_warp(lane, epi_smem + static_cast<size_t>(kEpiWarps) * kEpiWarpBytes);
  } else if (warp >= 4) {
    // ===================== consumers: MMA + epilogue =====================
    const int cg = (warp >> 2) - 1;     // consumer warpgroup: rows [64 cg, 64 cg + 64) of the tile
    const int ew = warp - 4;            // consumer warp: rows [16 ew, 16 ew + 16)
    const bool releaser = (threadIdx.x & 127) == 0;
    auto release = [&](int s) {
      if (!releaser) return;
      if (kCluster > 1) {
        mbar_arrive_cluster(&empty_bar[s], 0);
        mbar_arrive_cluster(&empty_bar[s], 1);
      } else {
        ptx::mbar_arrive(&empty_bar[s]);
      }
    };
    float d[kAccRegs];
    int stage = 0;
    uint32_t phase = 0;
    for (int item = first_item; item < num_items; item += item_stride) {
      const int tile = item * kCluster + crank;
      int m_blk, n_blk;
      policy.coords(tile, &m_blk, &n_blk);
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);  // TMA bytes landed
        const uint32_t sa = ptx::smem_u32(smem + static_cast<size_t>(stage) * kStageBytesT);
        wgmma_fence_operand(d);
        wgmma_fence();
        wgmma_kblock(d, sa + static_cast<uint32_t>(cg) * (kABytes / kConsumers), sa + kABytes, kb != 0);
        wgmma_commit();
        wgmma_wait<1>();                 // the previous k-block's MMAs are done: its stage may be refilled
        wgmma_fence_operand(d);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == kStagesT) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(d);
      if (prev >= 0) release(prev);
      policy.epilogue(d, epi_smem, m_blk * kBM, n_blk * kBN, ew, lane);
    }
  }

  __syncthreads();
  // A CTA of a pair must not retire while its partner can still multicast into it or arrive on its barriers.
  if (kCluster > 1) cluster_sync_all();
  policy.finish();
}

inline PFN_cuTensorMapEncodeTiled gemm_tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(p);
    (void)cudaGetLastError();
  });
  HPCP_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is not available");
  return fn;
}

// 2-D fp32 / bf16 [rows, cols] row-major tensor with a [16 rows x 128 bytes] SWIZZLE_128B box: the destination of
// the TMA epilogues (cp.async.bulk.tensor.2d store, cp.reduce.async.bulk.tensor.2d ... .add).
inline CUtensorMap make_c_tile_map(const void* base, int rows, int cols, bool bf16) {
  CUtensorMap map;
  const size_t elem = bf16 ? 2 : 4;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * elem};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / elem), static_cast<cuuint32_t>(kEpiRows)};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult r = gemm_tensor_map_encoder()(
      &map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims,
      strides, box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
      CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HPCP_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (C tile map) failed with code " + std::to_string(r));
  return map;
}

// 2-D bf16 [rows, k] K-major tensor with a [box_rows x 64] SWIZZLE_128B box.
inline CUtensorMap make_kmajor_map(const void* base, int rows, int k, int box_rows) {
  CUtensorMap map;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(k) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kBK), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult r = gemm_tensor_map_encoder()(
      &map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, elem_strides,
      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  HPCP_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " + std::to_string(r));
  return map;
}

}  // namespace umma
}  // namespace hpcp
