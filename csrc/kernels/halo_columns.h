// Which thread of which CTA handles which float4 column of a K-halo row, as plain integer functions shared by the
// device code (halo_stencil.cu) and the host (bindings -> tests/test_halo_column_map.py checks on a machine without a
// GPU that every float4 of a launch's column range has exactly one owner and nothing outside it has one).
//
// The map depends on the geometry alone, never on the rank or the step: CTA c owns the same column tiles on every
// rank, and thread t of CTA c the same float4s in every step.  So a thread only ever reads what it wrote itself in the
// previous step or what a neighbour's CTA c wrote before publishing its step word.
#pragma once

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HPCP_HD __host__ __device__ __forceinline__
#else
#define HPCP_HD inline
#endif

namespace hpcp {

constexpr int kHaloThreads = 512;  // threads per CTA of the stencil kernel

struct HaloColumns {
  uint64_t row_vec;                // float4 per row
  uint32_t tile_vec;               // float4 per column tile
  uint64_t tile_begin, tile_end;   // column tiles [begin, end) of this launch
  uint32_t ctas, threads;
};

// Column tiles of CTA c: tile_begin + c + jj * ctas for jj < halo_cta_tiles.
HPCP_HD uint64_t halo_cta_tiles(const HaloColumns& g, uint32_t cta) {
  const uint64_t n = g.tile_end - g.tile_begin;
  return n > cta ? (n - cta + g.ctas - 1) / g.ctas : 0;
}
// First float4 of the jj-th tile of CTA c; the tile ends at halo_tile_end.  Thread t handles first + t + k * threads.
HPCP_HD uint64_t halo_tile_first(const HaloColumns& g, uint32_t cta, uint64_t jj) {
  return (g.tile_begin + cta + jj * g.ctas) * g.tile_vec;
}
HPCP_HD uint64_t halo_tile_end(const HaloColumns& g, uint64_t first) {
  return first + g.tile_vec < g.row_vec ? first + g.tile_vec : g.row_vec;
}

// Owner of float4 column v: false when the launch does not touch it.
HPCP_HD bool halo_column_owner(const HaloColumns& g, uint64_t v, uint32_t* cta, uint32_t* thread) {
  const uint64_t tile = v / g.tile_vec;
  if (v >= g.row_vec || tile < g.tile_begin || tile >= g.tile_end) return false;
  *cta = static_cast<uint32_t>((tile - g.tile_begin) % g.ctas);
  *thread = static_cast<uint32_t>((v - tile * g.tile_vec) % g.threads);
  return true;
}

}  // namespace hpcp
