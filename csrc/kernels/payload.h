// Payload hash shared by the device fills and checks (p2p.cu, fused_triad_put.cu) and the host-only paths of the
// CLIs: a seeded bijection of the element index, so a word that lands at another index, or comes from another seed,
// almost surely has another value.  The Python twin is hpc_patterns_b200.ops.p2p.pattern_reference.
#pragma once

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define HPCP_HD __host__ __device__ __forceinline__
#else
#define HPCP_HD inline
#endif

namespace hpcp {

HPCP_HD uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// word[i] = mix32(i*2654435761 ^ seed) (↔ fill_randomly, p2p/peer2pear.cpp:8-17); i is taken modulo 2^32.
HPCP_HD uint32_t pattern_word(size_t i, uint32_t seed) {
  return mix32(static_cast<uint32_t>(i) * 2654435761u ^ seed);
}

// Triad inputs of rank r: one pattern word per element, b = its low 10 bits, c = the next 3 (small integers, so
// b + s*c is exact for s = 3).  Unlike a pattern that repeats every 1024 elements, a tile stored at another tile's
// offset, or a stage that still holds an older tile, changes almost every element.
constexpr uint32_t kTriadSeed = 0x7a1ad000u;
HPCP_HD uint32_t triad_word(size_t i, int rank) { return pattern_word(i, kTriadSeed + static_cast<uint32_t>(rank)); }
HPCP_HD uint32_t triad_b_bits(uint32_t w) { return w & 1023u; }
HPCP_HD uint32_t triad_c_bits(uint32_t w) { return (w >> 10) & 7u; }

}  // namespace hpcp
