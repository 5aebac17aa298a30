// Tile and gather-piece orderings of the tensor-core kernels as plain integer functions, shared by the device
// code (wgmma.cuh, gemm_collective.cu) and the host (bindings -> tests/test_tile_order.py checks that every order
// is a bijection, that CTA pairs get vertically adjacent tiles and that the gather covers every remote byte
// exactly once — on a machine without a GPU).
#pragma once

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HPCP_HD __host__ __device__ __forceinline__
#else
#define HPCP_HD inline
#endif

namespace hpcp {
namespace umma {

// Tile rasterisation: groups of kGroupM tile-rows, m fastest inside a group, so the ~132 tiles that
// are in flight at any time cover a near-square block of C (8 x ~17 tiles): fewer distinct A/B
// panels per k-step than row-major order -> less HBM traffic once A and B exceed the 50 MB L2.
constexpr int kGroupM = 8;
HPCP_HD void tile_coords(int tile, int tiles_m, int tiles_n, int* m_blk, int* n_blk) {
  const int group_size = kGroupM * tiles_n;
  const int group = tile / group_size;
  const int first_m = group * kGroupM;
  const int gm = tiles_m - first_m < kGroupM ? tiles_m - first_m : kGroupM;
  const int in_group = tile - group * group_size;
  *m_blk = first_m + in_group % gm;
  *n_blk = in_group / gm;
}

// Shard-major rasterisation: P groups of (M/P x N) tiles; group i of rank r is the shard of rank (r+first+i) % P,
// the grouped order above inside a shard.
HPCP_HD void shard_coords(int tile, int rank, int world, int first, int shard_tiles_m, int tiles_n, int* m_blk,
                          int* n_blk) {
  const int per_shard = shard_tiles_m * tiles_n;
  const int i = tile / per_shard;
  const int owner = (rank + first + i) % world;
  int mb;
  tile_coords(tile - i * per_shard, shard_tiles_m, tiles_n, &mb, n_blk);
  *m_blk = owner * shard_tiles_m + mb;
}

// All-gather -> GEMM: the (world-1) * shard_tiles_m * chunks_per_block remote pieces in the order the tile loop
// needs them (peer rank+1 first); piece c belongs to CTA c % grid.
struct GatherPiece {
  int peer;          // rank the piece is read from
  int m_blk;         // 128-row block of the gathered A it belongs to (its arrival counter)
  size_t src_off;    // byte offset inside the peer's row block
  size_t dst_off;    // byte offset inside the local gathered A
};
HPCP_HD GatherPiece gather_piece(size_t c, int rank, int world, int shard_tiles_m, uint32_t chunks_per_block,
                                 uint32_t chunk_bytes, size_t block_bytes) {
  const size_t per_peer = static_cast<size_t>(shard_tiles_m) * chunks_per_block;
  const int i = static_cast<int>(c / per_peer);  // i-th peer after me
  const size_t in_peer = c - i * per_peer;
  GatherPiece p;
  p.peer = (rank + 1 + i) % world;
  const size_t blk = in_peer / chunks_per_block;  // 128-row block inside the peer's rows
  p.src_off = blk * block_bytes + (in_peer - blk * chunks_per_block) * chunk_bytes;
  p.m_blk = p.peer * shard_tiles_m + static_cast<int>(blk);
  p.dst_off = static_cast<size_t>(p.peer) * shard_tiles_m * block_bytes + p.src_off;
  return p;
}

}  // namespace umma
}  // namespace hpcp
