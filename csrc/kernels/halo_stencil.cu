// K-halo: slab-decomposed 3-point stencil fused with its halo exchange — the suite's flagship.
//
// The reference's only communication loop is "kernel; wait; MPI_Send/Recv with both ring
// neighbours; wait; swap; kernel" (allreduce-mpi-sycl.cpp:167-181: Accumulate().wait(),
// SendRecvRing(VA -> right, VB <- left), swap, Accumulate().wait()): every step's compute
// consumes what the previous step received, and nothing overlaps.  K-halo is that dependency
// structure as an H100 kernel.  The global field is [world * rows][row_elems] floats, periodic in
// the row dimension and split into slabs of `rows` rows per GPU (one row = one message of the
// p2p benchmark, 188 743 680 B by default, p2p/peer2pear.cpp:115-116).  One step is the stream
// triad  a = b + s * c  with  b = alpha * u[r],  c = u[r-1] + u[r+1]:
//
//     u'[r][j] = alpha * u[r][j] + s * (u[r-1][j] + u[r+1][j])
//
// Row -1 is the left neighbour's last row and row `rows` the right neighbour's first row of the
// SAME step's input: the halo.  Two forms of the exchange, both inside the stencil kernel:
//   pull  the kernel reads the neighbours' boundary rows straight out of their field over NVLink
//         (128-bit loads from a peer-mapped address).  No halo buffer exists, the halo costs no HBM
//         write and no HBM read on the consumer.
//   push  the kernel stores its freshly computed boundary rows into halo buffers on the neighbours
//         (128-bit stores to a peer-mapped address) next to the local store, from the same registers.
// `none` reads local halo buffers and talks to nobody: the compute kernel of the stock arm
// (kernel -> cudaMemcpyAsync / NCCL send+recv -> host wait), which models/halo.py times next to it.
//
// Work split (halo_columns.h).  A CTA owns column tiles j = blockIdx.x + k * gridDim.x of EVERY row, and thread t of
// the CTA the float4 columns t, t + kHaloThreads, ... of each of its tiles.  A thread loads all R + 2 input rows of
// one of its columns into registers, computes the R outputs and stores them: a plain 128-bit ld/st stream, the engine
// of the card's fastest copy, with no shared memory and no intra-CTA hand-off.  Because the map does not depend on the
// rank or the step, a thread only reads what it wrote itself in the previous step (its own rows, and at N = 1 both
// halos) or what a neighbour's CTA c published, so the only cross-CTA dependency of step g+1 is "CTA c of my two
// neighbours finished step g".  That is one monotonic word per (neighbour, CTA):
//   * RAW  my step g reads the neighbour's u_g boundary tile / my halo[g&1]: written in its step g-1;
//   * WAR  my step g overwrites u[(g+1)&1] / the neighbour's halo[(g+1)&1]: last read in its step g-1.
// Both are "neighbour's CTA c completed step g-1", i.e. flag >= g.  Thread 0 waits for both words, then
// __syncthreads(); after the CTA's last store of the step, __syncthreads(), fence.acq_rel.sys and st.release.sys of
// g+1 to both neighbours (signal.cuh).  In pull and push mode the CTAs also pace each other through a rank-local
// count of finished tiles (see the kernel), so that they stay within one wave of tiles.  So K steps run in ONE launch with no grid barrier, no host sync and no
// per-step launch (`steps` > 1), or one launch per step (`steps` == 1) with the same words carrying the dependency
// across launches.  Loads are never `.nc`: the kernel reads data that it or a peer wrote earlier in the same launch.
//
// Load order of a column: boundary rows first — own row R-1, up halo, own row 0, down halo, then rows 1 .. R-2
// (R = 1: row 0, up, down).  Every boundary row is read twice per step by somebody: by its owner as a centre row and
// by a neighbour as its halo (at N = 1 the neighbour is the rank itself, so up halo = own row R-1 and down halo = own
// row 0).  With this order the two reads of a row sit next to each other, and since ranks run CTA by CTA in near
// lock-step the second one is served from L2: a step moves 2 * rows rows through HBM, not 2 * rows + 2.  L2 policy by
// role: interior-row loads and the local stores stream with evict_first, boundary-row loads keep the default policy so
// that the second read finds them; nothing is allocated in L1.  The interior rows are loaded kHaloChunk at a time
// ahead of their use, so at R = 8 all ten loads of a column are in flight at once.
#include "api.h"

#include <algorithm>
#include <mutex>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "halo_columns.h"

namespace hpcp {

namespace {

constexpr int kHaloCtasPerSm = 2;  // 1024 threads per SM: <= 64 registers per thread
constexpr int kHaloChunk = 6;      // interior rows loaded ahead of their use
constexpr int kHaloDefaultTileKb = 16;

struct HaloParams {
  float4* u[2];
  const float4* up_src[2];  // row -1 of step parity p: pull = left neighbour's last row, else halo_lo[p]
  const float4* dn_src[2];  // row `rows`:              pull = right neighbour's row 0,   else halo_hi[p]
  float4* put_first[2];     // push: where my new row 0 goes on the left neighbour (its halo_hi[p])
  float4* put_last[2];      // push: where my new last row goes on the right neighbour (its halo_lo[p])
  // Flag arrays, one 32-byte sector per CTA (index blockIdx.x * kHaloFlagWords):
  const uint32_t* wait_lo;  // local, written by the left neighbour's CTAs
  const uint32_t* wait_hi;  // local, written by the right neighbour's CTAs
  uint32_t* signal_lo;      // on the left neighbour (its wait_hi array)
  uint32_t* signal_hi;      // on the right neighbour (its wait_lo array)
  uint32_t* pace;           // local: column tiles of this flag set finished on this rank, counting up forever
  int rows;
  HaloColumns cols;
  float alpha, s;
  uint32_t step_base;
  int steps;
  uint64_t timeout_ns;
  uint32_t* status;
};

__device__ __forceinline__ float stencil1(float up, float ce, float dn, float alpha, float s) {
  // Explicitly rounded, never contracted: bit-identical to `alpha * u + s * (up + dn)` evaluated
  // operation by operation in fp32 (the PyTorch reference of the tests).
  return __fadd_rn(__fmul_rn(alpha, ce), __fmul_rn(s, __fadd_rn(up, dn)));
}
__device__ __forceinline__ float4 stencil4(const float4& up, const float4& ce, const float4& dn, float alpha,
                                           float s) {
  return make_float4(stencil1(up.x, ce.x, dn.x, alpha, s), stencil1(up.y, ce.y, dn.y, alpha, s),
                     stencil1(up.z, ce.z, dn.z, alpha, s), stencil1(up.w, ce.w, dn.w, alpha, s));
}

// 128-bit accesses of the stencil, all L1::no_allocate and never `.nc`.
__device__ __forceinline__ float4 ld_keep(const float4* p) {  // boundary rows: read again right after, from L2
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_stream(const float4* p, uint64_t policy) {  // interior rows: read once
  float4 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p), "l"(policy)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream(float4* p, const float4& v, uint64_t policy) {  // local field
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void st_put(float4* p, const float4& v) {  // push: the neighbour's halo buffer
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// One step of float4 column v: loads in boundary-first order, outputs rows 0 .. R-1 in order.
template <int kMode>
__device__ __forceinline__ void halo_column(const HaloParams& p, int in, uint64_t v) {
  const uint64_t evict_first = ptx::l2_policy_evict_first();
  const int R = p.rows;
  const uint64_t rv = p.cols.row_vec;
  const float alpha = p.alpha, s = p.s;
  const float4* uin = p.u[in] + v;
  float4* uout = p.u[in ^ 1] + v;
  auto store = [&](int r, const float4& x) {
    st_stream(uout + static_cast<uint64_t>(r) * rv, x, evict_first);
    if (kMode == 2) {
      if (r == 0) st_put(p.put_first[in ^ 1] + v, x);
      if (r == R - 1) st_put(p.put_last[in ^ 1] + v, x);
    }
  };
  const float4 last = ld_keep(uin + static_cast<uint64_t>(R - 1) * rv);
  float4 prev = ld_keep(p.up_src[in] + v);
  if (R == 1) {
    store(0, stencil4(prev, last, ld_keep(p.dn_src[in] + v), alpha, s));
    return;
  }
  float4 cur = ld_keep(uin);
  const float4 dn = ld_keep(p.dn_src[in] + v);
  for (int base = 1; base < R - 1; base += kHaloChunk) {  // interior rows: row base-1 .. base+kHaloChunk-2 out
    float4 w[kHaloChunk];
#pragma unroll
    for (int i = 0; i < kHaloChunk; ++i)
      if (base + i < R - 1) w[i] = ld_stream(uin + static_cast<uint64_t>(base + i) * rv, evict_first);
#pragma unroll
    for (int i = 0; i < kHaloChunk; ++i) {
      if (base + i < R - 1) {
        store(base + i - 1, stencil4(prev, cur, w[i], alpha, s));
        prev = cur;
        cur = w[i];
      }
    }
  }
  store(R - 2, stencil4(prev, cur, last, alpha, s));
  store(R - 1, stencil4(cur, last, dn, alpha, s));
}

// kMode: 0 none, 1 pull, 2 push.
template <int kMode>
__global__ void __launch_bounds__(kHaloThreads, kHaloCtasPerSm) halo_stencil_kernel(const HaloParams p) {
  __shared__ int abort_w;
  const uint32_t ntiles = static_cast<uint32_t>(halo_cta_tiles(p.cols, blockIdx.x));  // < 2^32 float4 per row
  if (ntiles == 0) return;  // same geometry on every rank: nobody waits for this CTA index
  for (int si = 0; si < p.steps; ++si) {
    const uint32_t g = p.step_base + static_cast<uint32_t>(si);
    const int in = static_cast<int>(g & 1u);
    for (uint32_t jj = 0; jj < ntiles; ++jj) {
      if (kMode != 0) {
        // Tile jj of step g is ticket t = g * n + jj * G + c of this rank and flag set (dense over the n tiles of a
        // step, in row order within a step).  Besides the neighbour words at the start of a step, the CTA waits until
        // at least t - G tickets of this rank are finished: CTAs that run ahead are held to one wave of tiles, so the
        // CTAs stream through a compact stretch of the rows together, as one-shot grids do.  On an H100 that is
        // worth ~2 % of HBM throughput over free-running CTAs.  The wait only ever needs earlier tickets (or the
        // neighbours' earlier steps), so it cannot deadlock; it is not needed for correctness.
        if (threadIdx.x == 0) {
          const uint32_t n = static_cast<uint32_t>(p.cols.tile_end - p.cols.tile_begin);
          const uint32_t ticket = g * n + jj * gridDim.x + blockIdx.x;
          abort_w = !((jj != 0 || (wait_epoch(p.wait_lo + blockIdx.x * kHaloFlagWords, g, p.timeout_ns, p.status) &&
                                   wait_epoch(p.wait_hi + blockIdx.x * kHaloFlagWords, g, p.timeout_ns, p.status))) &&
                      wait_epoch(p.pace, ticket - gridDim.x, p.timeout_ns, p.status));
        }
        __syncthreads();
        if (abort_w) return;
      }
      const uint64_t first = halo_tile_first(p.cols, blockIdx.x, jj);
      const uint64_t end = halo_tile_end(p.cols, first);
      for (uint64_t v = first + threadIdx.x; v < end; v += kHaloThreads) halo_column<kMode>(p, in, v);
      if (kMode != 0) {
        __syncthreads();  // every store of the tile (local field and, in push mode, the peers' halos)
        if (threadIdx.x == 0) {
          ptx::red_release_gpu_add(p.pace, 1u);
          if (jj + 1 == ntiles) {  // the step's last tile: publish the step to both neighbours
            ptx::fence_acq_rel_sys();
            ptx::st_release_sys(p.signal_hi + blockIdx.x * kHaloFlagWords, g + 1u);
            ptx::st_release_sys(p.signal_lo + blockIdx.x * kHaloFlagWords, g + 1u);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------- field values ----
// u0(global row, column): a hash folded to [-32, 32) with 10 fractional bits, reproducible on the host
// (models/halo.py::initial_field).
__device__ __forceinline__ float halo_u0(uint32_t grow, uint64_t j) {
  const uint32_t jl = static_cast<uint32_t>(j);
  const uint32_t h = (grow * 2654435761u) ^ (jl * 40503u + (jl >> 11));
  return static_cast<float>(static_cast<int>(h & 0xFFFFu) - 32768) * (1.0f / 1024.0f);
}

__global__ void halo_init_kernel(float* __restrict__ u, float* __restrict__ halo_lo, float* __restrict__ halo_hi,
                                 int rows, size_t row_elems, int rank, int world) {
  const uint32_t grows = static_cast<uint32_t>(rows) * world;
  const uint32_t first = static_cast<uint32_t>(rank) * rows;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < row_elems; j += stride) {
    for (int r = 0; r < rows; ++r) u[static_cast<size_t>(r) * row_elems + j] = halo_u0(first + r, j);
    if (halo_lo != nullptr) halo_lo[j] = halo_u0((first + grows - 1) % grows, j);
    if (halo_hi != nullptr) halo_hi[j] = halo_u0((first + rows) % grows, j);
  }
}

// Independent check from the closed-form initial field: every thread owns one column of the GLOBAL
// field (all world * rows rows), advances it `steps` times with the periodic stencil in the kernel's
// operation order and compares this rank's rows exactly.
constexpr int kHaloMaxGlobalRows = 128;
__global__ void halo_verify_init_kernel(const float* __restrict__ u, int rows, size_t row_elems, int rank, int world,
                                        uint32_t steps, float alpha, float s, unsigned long long* mismatch_count) {
  const int G = rows * world;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  float v[kHaloMaxGlobalRows];
  for (size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < row_elems; j += stride) {
    for (int g = 0; g < G; ++g) v[g] = halo_u0(static_cast<uint32_t>(g), j);
    for (uint32_t k = 0; k < steps; ++k) {
      const float first = v[0];
      float prev = v[G - 1];
      for (int g = 0; g < G; ++g) {
        const float cur = v[g];
        const float next = g + 1 < G ? v[g + 1] : first;
        v[g] = stencil1(prev, cur, next, alpha, s);
        prev = cur;
      }
    }
    for (int r = 0; r < rows; ++r) bad += (__ldcg(u + static_cast<size_t>(r) * row_elems + j) != v[rank * rows + r]);
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatch_count, bad);
}

// Check of ONE step through an independent data path: plain (coherent) vector loads of the step's input,
// including the neighbours' boundary rows wherever they live (peer-mapped field or local halo buffer).
__global__ void halo_verify_step_kernel(const float* __restrict__ u_new, const float* __restrict__ u_old,
                                        const float* __restrict__ up_row, const float* __restrict__ dn_row, int rows,
                                        size_t row_elems, float alpha, float s, unsigned long long* mismatch_count) {
  const size_t nvec = row_elems / 4;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  auto ld = [](const float* base, size_t v) {
    const uint4 w = ptx::ld_peer_v4(reinterpret_cast<const uint4*>(base) + v);
    return make_float4(__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), __uint_as_float(w.w));
  };
  for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    float4 up = ld(up_row, v);
    float4 ce = ld(u_old, v);
    for (int r = 0; r < rows; ++r) {
      const float4 dn = r + 1 < rows ? ld(u_old + static_cast<size_t>(r + 1) * row_elems, v) : ld(dn_row, v);
      const float4 want = stencil4(up, ce, dn, alpha, s);
      const float4 got = ld(u_new + static_cast<size_t>(r) * row_elems, v);
      bad += (got.x != want.x) + (got.y != want.y) + (got.z != want.z) + (got.w != want.w);
      up = ce;
      ce = dn;
    }
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatch_count, bad);
}

struct HaloGeometry {
  uint32_t tile_bytes;
  int ctas;
};

template <int kMode>
int occupancy_of() {
  // One occupancy query per (mode, device), not per launch (per-step launches come here K times).
  static std::mutex mu;
  static int per_sm[64] = {0};
  int device = 0;
  HPCP_CUDA(cudaGetDevice(&device));
  std::lock_guard<std::mutex> lk(mu);
  if (device < 0 || device >= 64 || per_sm[device] == 0) {
    int n = 0;
    HPCP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, halo_stencil_kernel<kMode>, kHaloThreads, 0));
    if (device < 0 || device >= 64) return n;
    per_sm[device] = n;
  }
  return per_sm[device];
}

HaloGeometry halo_geometry(size_t row_bytes, const HaloTuning& tune, HaloMode mode, int device) {
  HaloGeometry g;
  HPCP_REQUIRE(tune.tile_kb >= 0 && tune.tile_kb <= 1024, "halo_stencil: tile_kb in 1 .. 1024 (0 -> 16)");
  g.tile_bytes = static_cast<uint32_t>((tune.tile_kb > 0 ? tune.tile_kb : kHaloDefaultTileKb) * 1024);
  const int sms = device_sm_count(device);
  int per_sm = 1;
  // Co-residency: a persistent multi-step launch spins on neighbour words, so every CTA must be resident.
  switch (mode) {
    case HaloMode::kNone: per_sm = occupancy_of<0>(); break;
    case HaloMode::kPull: per_sm = occupancy_of<1>(); break;
    case HaloMode::kPush: per_sm = occupancy_of<2>(); break;
  }
  HPCP_REQUIRE(per_sm >= 1, "halo_stencil: kernel does not fit on an SM");
  const size_t tiles = (row_bytes + g.tile_bytes - 1) / g.tile_bytes;
  const int resident = std::min(sms * std::min(per_sm, kHaloCtasPerSm), kHaloMaxCtas);  // one step word per CTA
  const int want = tune.ctas > 0 ? std::min(tune.ctas, resident) : resident;
  g.ctas = static_cast<int>(std::max<size_t>(1, std::min<size_t>(tiles, static_cast<size_t>(want))));
  HPCP_REQUIRE(g.ctas <= kHaloMaxCtas, "halo_stencil: more CTAs than flag words");
  return g;
}

}  // namespace

int halo_stencil_ctas(size_t row_elems, const HaloTuning& tune, HaloMode mode, int device) {
  return halo_geometry(row_elems * sizeof(float), tune, mode, device).ctas;
}

int launch_halo_stencil(const HaloStencilArgs& a, HaloMode mode, const HaloTuning& tune, int device,
                        cudaStream_t stream) {
  HPCP_REQUIRE(a.rows >= 1 && a.row_elems > 0 && a.row_elems % 4 == 0,
               "halo_stencil: rows >= 1 and row_elems a positive multiple of 4");
  HPCP_REQUIRE(a.steps >= 1, "halo_stencil: steps >= 1");
  HPCP_REQUIRE(a.u[0] != nullptr && a.u[1] != nullptr, "halo_stencil: both field buffers are needed");
  const size_t row_bytes = a.row_elems * sizeof(float);
  const HaloGeometry g = halo_geometry(row_bytes, tune, mode, device);
  const int ctas = g.ctas;
  const size_t tiles_per_row = (row_bytes + g.tile_bytes - 1) / g.tile_bytes;
  HaloParams p{};
  for (int q = 0; q < 2; ++q) {
    p.u[q] = reinterpret_cast<float4*>(a.u[q]);
    if (mode == HaloMode::kPull) {
      HPCP_REQUIRE(a.left_u[q] != nullptr && a.right_u[q] != nullptr, "halo_stencil: pull needs the neighbours' fields");
      p.up_src[q] = reinterpret_cast<const float4*>(a.left_u[q] + static_cast<size_t>(a.rows - 1) * a.row_elems);
      p.dn_src[q] = reinterpret_cast<const float4*>(a.right_u[q]);
    } else {
      HPCP_REQUIRE(a.halo_lo[q] != nullptr && a.halo_hi[q] != nullptr, "halo_stencil: halo buffers are needed");
      p.up_src[q] = reinterpret_cast<const float4*>(a.halo_lo[q]);
      p.dn_src[q] = reinterpret_cast<const float4*>(a.halo_hi[q]);
    }
    if (mode == HaloMode::kPush) {
      HPCP_REQUIRE(a.left_halo_hi[q] != nullptr && a.right_halo_lo[q] != nullptr,
                   "halo_stencil: push needs the neighbours' halo buffers");
      p.put_first[q] = reinterpret_cast<float4*>(a.left_halo_hi[q]);
      p.put_last[q] = reinterpret_cast<float4*>(a.right_halo_lo[q]);
    }
  }
  if (mode != HaloMode::kNone) {
    HPCP_REQUIRE(a.flags_local != nullptr && a.flags_left != nullptr && a.flags_right != nullptr,
                 "halo_stencil: neighbour flag words are needed");
    HPCP_REQUIRE(a.flag_set >= 0 && a.flag_set < kHaloFlagSets, "halo_stencil: flag_set out of range");
  }
  p.rows = a.rows;
  p.cols.row_vec = a.row_elems / 4;
  p.cols.tile_vec = g.tile_bytes / 16;
  p.cols.tile_begin = a.tile_begin;
  p.cols.tile_end = a.tile_end == 0 ? tiles_per_row : a.tile_end;
  HPCP_REQUIRE(p.cols.tile_begin < p.cols.tile_end && p.cols.tile_end <= tiles_per_row,
               "halo_stencil: bad column-tile range");
  p.cols.ctas = static_cast<uint32_t>(ctas);
  p.cols.threads = kHaloThreads;
  p.alpha = a.alpha;
  p.s = a.s;
  p.step_base = a.step_base;
  p.steps = a.steps;
  p.timeout_ns = a.timeout_ns;
  p.status = a.status;
  // Flag words: one 32-byte sector per (flag set, side, CTA); the kernel adds blockIdx.x * kHaloFlagWords.
  const size_t set_words = static_cast<size_t>(a.flag_set) * 2 * kHaloMaxCtas * kHaloFlagWords;
  const size_t side_words = static_cast<size_t>(kHaloMaxCtas) * kHaloFlagWords;
  auto launch = [&](auto kernel) { kernel<<<ctas, kHaloThreads, 0, stream>>>(p); };
  if (mode != HaloMode::kNone) {
    p.wait_lo = a.flags_local + set_words;
    p.wait_hi = a.flags_local + set_words + side_words;
    p.signal_lo = a.flags_left + set_words + side_words;  // I am the right neighbour of my left neighbour
    p.signal_hi = a.flags_right + set_words;              // and the left neighbour of my right neighbour
    p.pace = a.flags_local + set_words + 1;               // word 1 of CTA 0's sector of the wait_lo side (unused)
  }
  switch (mode) {
    case HaloMode::kNone: launch(halo_stencil_kernel<0>); break;
    case HaloMode::kPull: launch(halo_stencil_kernel<1>); break;
    case HaloMode::kPush: launch(halo_stencil_kernel<2>); break;
  }
  HPCP_CUDA(cudaGetLastError());
  return ctas;
}

void launch_halo_init(float* u, float* halo_lo, float* halo_hi, int rows, size_t row_elems, int rank, int world,
                      cudaStream_t stream) {
  const int threads = 256;
  const int ctas = static_cast<int>(std::min<size_t>((row_elems + threads - 1) / threads, 132 * 8));
  halo_init_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(u, halo_lo, halo_hi, rows, row_elems, rank, world);
  HPCP_CUDA(cudaGetLastError());
}

void launch_halo_verify_from_init(const float* u, int rows, size_t row_elems, int rank, int world, uint32_t steps,
                                  float alpha, float s, unsigned long long* mismatch_count, cudaStream_t stream) {
  HPCP_REQUIRE(rows * world <= kHaloMaxGlobalRows, "halo verify: world * rows exceeds 128 global rows");
  const int threads = 128;
  const int ctas = static_cast<int>(std::min<size_t>((row_elems + threads - 1) / threads, 132 * 16));
  halo_verify_init_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(u, rows, row_elems, rank, world, steps, alpha, s,
                                                                    mismatch_count);
  HPCP_CUDA(cudaGetLastError());
}

void launch_halo_verify_step(const float* u_new, const float* u_old, const float* up_row, const float* dn_row,
                             int rows, size_t row_elems, float alpha, float s, unsigned long long* mismatch_count,
                             cudaStream_t stream) {
  const int threads = 256;
  const int ctas = static_cast<int>(std::min<size_t>((row_elems / 4 + threads - 1) / threads, 132 * 8));
  halo_verify_step_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(u_new, u_old, up_row, dn_row, rows, row_elems,
                                                                    alpha, s, mismatch_count);
  HPCP_CUDA(cudaGetLastError());
}

}  // namespace hpcp
