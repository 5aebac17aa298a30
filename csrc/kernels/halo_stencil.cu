// K-halo: slab-decomposed 3-point stencil fused with its halo exchange — the suite's flagship.
//
// The reference's only communication loop is "kernel; wait; MPI_Send/Recv with both ring
// neighbours; wait; swap; kernel" (allreduce-mpi-sycl.cpp:167-181: Accumulate().wait(),
// SendRecvRing(VA -> right, VB <- left), swap, Accumulate().wait()): every step's compute
// consumes what the previous step received, and nothing overlaps.  K-halo is that dependency
// structure as an H100 kernel.  The global field is [world * rows][row_elems] elements of one field type (float by
// default; double, bfloat16 and half share the same body through a 16-byte vector type, below), periodic in
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
#include <cstring>
#include <map>
#include <mutex>
#include <utility>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "halo_columns.h"
#include "halo_field.h"

namespace hpcp {

namespace {

constexpr int kHaloCtasPerSm = 2;  // 1024 threads per SM: <= 64 registers per thread
constexpr int kHaloChunk = 6;      // interior rows loaded ahead of their use (fp32, fp64; see Pair16Vec)
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
// The same four accesses on raw 16-byte words, for the double and 16-bit fields.
__device__ __forceinline__ uint4 ld_keep(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_stream(const uint4* p, uint64_t policy) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p), "l"(policy)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream(uint4* p, const uint4& v, uint64_t policy) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void st_put(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ------------------------------------------------------- 16-byte vectors ----
// A "16-byte vector of T" is what one thread moves per row and column: its raw register type (`Raw`), the interior
// rows it keeps in flight (`kChunk`), the stencil on it, and the two helpers of the step check.  Every field type computes one step per element as: widen the three
// inputs exactly to the compute type (fp32, or fp64 for double), alpha*u + s*(up + dn) one rounded operation at a time,
// never contracted, then round once to T (round-to-nearest-even, subnormals kept).  alpha and s are fp32 values.
__device__ __forceinline__ double stencil1(double up, double ce, double dn, float alpha, float s) {
  return __dadd_rn(__dmul_rn(static_cast<double>(alpha), ce), __dmul_rn(static_cast<double>(s), __dadd_rn(up, dn)));
}

// The rule of both halo checks: an element is wrong iff its bit pattern differs from the reference's, unless both are
// NaN (of any sign or payload: the GPU's and the host's canonical NaNs differ).  So a wrong sign of zero or a flushed
// subnormal is counted, and a NaN where a NaN is due is not.  `mag` clears the sign bit, `inf` is the infinity pattern.
template <class B>
__device__ __forceinline__ int bits_differ(B a, B b, B mag, B inf) {
  return a != b && !((a & mag) > inf && (b & mag) > inf);
}

// Element <-> compute type (FieldElem, halo_field.h), `differs` (the rule above), and a 32-bit word <-> a pair of
// 16-bit elements (element 2i in the low half).
template <class T>
struct Elem;
template <>
struct Elem<float> : FieldElem<float> {
  __device__ static __forceinline__ int differs(float a, float b) {
    return bits_differ<uint32_t>(__float_as_uint(a), __float_as_uint(b), 0x7FFFFFFFu, 0x7F800000u);
  }
};
template <>
struct Elem<double> : FieldElem<double> {
  __device__ static __forceinline__ int differs(double a, double b) {
    return bits_differ<uint64_t>(__double_as_longlong(a), __double_as_longlong(b), 0x7FFFFFFFFFFFFFFFull,
                                 0x7FF0000000000000ull);
  }
};
template <>
struct Elem<__nv_bfloat16> : FieldElem<__nv_bfloat16> {
  __device__ static __forceinline__ int differs(__nv_bfloat16 a, __nv_bfloat16 b) {
    return bits_differ<uint16_t>(__bfloat16_as_ushort(a), __bfloat16_as_ushort(b), 0x7FFFu, 0x7F80u);
  }
  __device__ static __forceinline__ __nv_bfloat16 from_half_word(uint32_t w) {  // the low 16 bits of w
    return __ushort_as_bfloat16(static_cast<unsigned short>(w));
  }
  __device__ static __forceinline__ float2 widen2(uint32_t w) {  // bf16 is the high half of an fp32: one op per lane
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
  }
  __device__ static __forceinline__ uint32_t narrow2(float2 f) {
    const __nv_bfloat162 h = __float22bfloat162_rn(f);
    uint32_t w;
    memcpy(&w, &h, 4);
    return w;
  }
};
template <>
struct Elem<__half> : FieldElem<__half> {
  __device__ static __forceinline__ int differs(__half a, __half b) {
    return bits_differ<uint16_t>(__half_as_ushort(a), __half_as_ushort(b), 0x7FFFu, 0x7C00u);
  }
  __device__ static __forceinline__ __half from_half_word(uint32_t w) {
    return __ushort_as_half(static_cast<unsigned short>(w));
  }
  __device__ static __forceinline__ float2 widen2(uint32_t w) {
    __half2 h;
    memcpy(&h, &w, 4);
    return __half22float2(h);
  }
  __device__ static __forceinline__ uint32_t narrow2(float2 f) {
    const __half2 h = __float22half2_rn(f);
    uint32_t w;
    memcpy(&w, &h, 4);
    return w;
  }
};

struct F32Vec {  // 4 lanes: the fp32 kernels' float4 code
  using Raw = float4;
  static constexpr int kChunk = kHaloChunk;
  __device__ static __forceinline__ Raw stencil(const Raw& up, const Raw& ce, const Raw& dn, float alpha, float s) {
    return stencil4(up, ce, dn, alpha, s);
  }
  __device__ static __forceinline__ Raw from_bits(const uint4& w) {
    return make_float4(__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), __uint_as_float(w.w));
  }
  __device__ static __forceinline__ int mismatches(const Raw& got, const Raw& want) {
    using E = Elem<float>;
    return E::differs(got.x, want.x) + E::differs(got.y, want.y) + E::differs(got.z, want.z) +
           E::differs(got.w, want.w);
  }
};

struct F64Vec {  // 2 lanes, each a pair of 32-bit words
  using Raw = uint4;
  static constexpr int kChunk = kHaloChunk;
  __device__ static __forceinline__ double lane(uint32_t lo, uint32_t hi) {
    return __hiloint2double(static_cast<int>(hi), static_cast<int>(lo));
  }
  __device__ static __forceinline__ Raw stencil(const Raw& up, const Raw& ce, const Raw& dn, float alpha, float s) {
    const double a = stencil1(lane(up.x, up.y), lane(ce.x, ce.y), lane(dn.x, dn.y), alpha, s);
    const double b = stencil1(lane(up.z, up.w), lane(ce.z, ce.w), lane(dn.z, dn.w), alpha, s);
    return make_uint4(static_cast<uint32_t>(__double2loint(a)), static_cast<uint32_t>(__double2hiint(a)),
                      static_cast<uint32_t>(__double2loint(b)), static_cast<uint32_t>(__double2hiint(b)));
  }
  __device__ static __forceinline__ Raw from_bits(const uint4& w) { return w; }
  __device__ static __forceinline__ int mismatches(const Raw& got, const Raw& want) {
    return Elem<double>::differs(lane(got.x, got.y), lane(want.x, want.y)) +
           Elem<double>::differs(lane(got.z, got.w), lane(want.z, want.w));
  }
};

template <class T>  // 8 lanes of __nv_bfloat16 or __half, converted one 32-bit pair at a time where it is used
struct Pair16Vec {
  using Raw = uint4;
  // With six interior rows in flight the lane conversions push ptxas past 64 registers (an 8-byte spill inside the
  // push kernel's column code); five fit.  At R = 8 that is nine of the ten loads of a column in flight at once.
  static constexpr int kChunk = 5;
  __device__ static __forceinline__ uint32_t pair(uint32_t up, uint32_t ce, uint32_t dn, float alpha, float s) {
    const float2 u = Elem<T>::widen2(up), c = Elem<T>::widen2(ce), d = Elem<T>::widen2(dn);
    return Elem<T>::narrow2(make_float2(stencil1(u.x, c.x, d.x, alpha, s), stencil1(u.y, c.y, d.y, alpha, s)));
  }
  __device__ static __forceinline__ Raw stencil(const Raw& up, const Raw& ce, const Raw& dn, float alpha, float s) {
    return make_uint4(pair(up.x, ce.x, dn.x, alpha, s), pair(up.y, ce.y, dn.y, alpha, s),
                      pair(up.z, ce.z, dn.z, alpha, s), pair(up.w, ce.w, dn.w, alpha, s));
  }
  __device__ static __forceinline__ Raw from_bits(const uint4& w) { return w; }
  __device__ static __forceinline__ int lanes_differ(uint32_t a, uint32_t b) {
    using E = Elem<T>;
    return E::differs(E::from_half_word(a), E::from_half_word(b)) +
           E::differs(E::from_half_word(a >> 16), E::from_half_word(b >> 16));
  }
  __device__ static __forceinline__ int mismatches(const Raw& got, const Raw& want) {
    return lanes_differ(got.x, want.x) + lanes_differ(got.y, want.y) + lanes_differ(got.z, want.z) +
           lanes_differ(got.w, want.w);
  }
};

template <class T>
struct VecOf;
template <>
struct VecOf<float> {
  using type = F32Vec;
};
template <>
struct VecOf<double> {
  using type = F64Vec;
};
template <>
struct VecOf<__nv_bfloat16> {
  using type = Pair16Vec<__nv_bfloat16>;
};
template <>
struct VecOf<__half> {
  using type = Pair16Vec<__half>;
};

// One step of 16-byte column v: loads in boundary-first order, outputs rows 0 .. R-1 in order.
template <class V, int kMode>
__device__ __forceinline__ void halo_column(const HaloParams& p, int in, uint64_t v) {
  using Raw = typename V::Raw;
  const uint64_t evict_first = ptx::l2_policy_evict_first();
  const int R = p.rows;
  const uint64_t rv = p.cols.row_vec;
  const float alpha = p.alpha, s = p.s;
  const Raw* uin = reinterpret_cast<const Raw*>(p.u[in]) + v;
  Raw* uout = reinterpret_cast<Raw*>(p.u[in ^ 1]) + v;
  auto store = [&](int r, const Raw& x) {
    st_stream(uout + static_cast<uint64_t>(r) * rv, x, evict_first);
    if (kMode == 2) {
      if (r == 0) st_put(reinterpret_cast<Raw*>(p.put_first[in ^ 1]) + v, x);
      if (r == R - 1) st_put(reinterpret_cast<Raw*>(p.put_last[in ^ 1]) + v, x);
    }
  };
  const Raw last = ld_keep(uin + static_cast<uint64_t>(R - 1) * rv);
  Raw prev = ld_keep(reinterpret_cast<const Raw*>(p.up_src[in]) + v);
  if (R == 1) {
    store(0, V::stencil(prev, last, ld_keep(reinterpret_cast<const Raw*>(p.dn_src[in]) + v), alpha, s));
    return;
  }
  Raw cur = ld_keep(uin);
  const Raw dn = ld_keep(reinterpret_cast<const Raw*>(p.dn_src[in]) + v);
  for (int base = 1; base < R - 1; base += V::kChunk) {  // interior rows: row base-1 .. base+V::kChunk-2 out
    Raw w[V::kChunk];
#pragma unroll
    for (int i = 0; i < V::kChunk; ++i)
      if (base + i < R - 1) w[i] = ld_stream(uin + static_cast<uint64_t>(base + i) * rv, evict_first);
#pragma unroll
    for (int i = 0; i < V::kChunk; ++i) {
      if (base + i < R - 1) {
        store(base + i - 1, V::stencil(prev, cur, w[i], alpha, s));
        prev = cur;
        cur = w[i];
      }
    }
  }
  store(R - 2, V::stencil(prev, cur, last, alpha, s));
  store(R - 1, V::stencil(cur, last, dn, alpha, s));
}

// The stencil kernel of every field type: T = float, double, __nv_bfloat16, __half.  kMode: 0 none, 1 pull, 2 push.
template <class T, int kMode>
__global__ void __launch_bounds__(kHaloThreads, kHaloCtasPerSm) halo_stencil_kernel(const HaloParams p) {
  using V = typename VecOf<T>::type;
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
      for (uint64_t v = first + threadIdx.x; v < end; v += kHaloThreads) halo_column<V, kMode>(p, in, v);
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
// The closed-form initial field u0 (halo_u0, halo_field.h), rounded to the field type.
template <class T>
__global__ void halo_init_kernel(T* __restrict__ u, T* __restrict__ halo_lo, T* __restrict__ halo_hi, int rows,
                                 size_t row_elems, int rank, int world) {
  const uint32_t grows = static_cast<uint32_t>(rows) * world;
  const uint32_t first = static_cast<uint32_t>(rank) * rows;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < row_elems; j += stride) {
    for (int r = 0; r < rows; ++r) u[static_cast<size_t>(r) * row_elems + j] = Elem<T>::narrow(halo_u0(first + r, j));
    if (halo_lo != nullptr) halo_lo[j] = Elem<T>::narrow(halo_u0((first + grows - 1) % grows, j));
    if (halo_hi != nullptr) halo_hi[j] = Elem<T>::narrow(halo_u0((first + rows) % grows, j));
  }
}

// Independent check from the closed-form initial field: every thread owns one column of the GLOBAL
// field (all world * rows rows), advances it `steps` times with the periodic stencil in the kernel's
// operation order and compares this rank's rows bit for bit (Elem<T>::differs).  The column is kept in the compute
// type, rounded to T after every step as the field is, so narrowing it back to T is exact.
template <class T>
__global__ void halo_verify_init_kernel(const T* __restrict__ u, int rows, size_t row_elems, int rank, int world,
                                        uint32_t steps, float alpha, float s, unsigned long long* mismatch_count) {
  using C = typename Elem<T>::Compute;
  const int G = rows * world;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  C v[kHaloMaxGlobalRows];
  for (size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < row_elems; j += stride) {
    for (int g = 0; g < G; ++g) v[g] = Elem<T>::widen(Elem<T>::narrow(halo_u0(static_cast<uint32_t>(g), j)));
    for (uint32_t k = 0; k < steps; ++k) {
      const C first = v[0];
      C prev = v[G - 1];
      for (int g = 0; g < G; ++g) {
        const C cur = v[g];
        const C next = g + 1 < G ? v[g + 1] : first;
        v[g] = Elem<T>::widen(Elem<T>::narrow(stencil1(prev, cur, next, alpha, s)));
        prev = cur;
      }
    }
    for (int r = 0; r < rows; ++r)
      bad += Elem<T>::differs(__ldcg(u + static_cast<size_t>(r) * row_elems + j), Elem<T>::narrow(v[rank * rows + r]));
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatch_count, bad);
}

// Check of ONE step through an independent data path: plain (coherent) vector loads of the step's input,
// including the neighbours' boundary rows wherever they live (peer-mapped field or local halo buffer).
template <class T>
__global__ void halo_verify_step_kernel(const T* __restrict__ u_new, const T* __restrict__ u_old,
                                        const T* __restrict__ up_row, const T* __restrict__ dn_row, int rows,
                                        size_t row_elems, float alpha, float s, unsigned long long* mismatch_count) {
  using V = typename VecOf<T>::type;
  using Raw = typename V::Raw;
  const size_t nvec = row_elems / (16 / sizeof(T));
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  auto ld = [](const T* base, size_t v) { return V::from_bits(ptx::ld_peer_v4(reinterpret_cast<const uint4*>(base) + v)); };
  for (size_t v = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    Raw up = ld(up_row, v);
    Raw ce = ld(u_old, v);
    for (int r = 0; r < rows; ++r) {
      const Raw dn = r + 1 < rows ? ld(u_old + static_cast<size_t>(r + 1) * row_elems, v) : ld(dn_row, v);
      const Raw want = V::stencil(up, ce, dn, alpha, s);
      const Raw got = ld(u_new + static_cast<size_t>(r) * row_elems, v);
      bad += V::mismatches(got, want);
      up = ce;
      ce = dn;
    }
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatch_count, bad);
}

using StencilKernel = void (*)(HaloParams);

// The stencil kernel of a field type and mode: the one place that maps (ElemType, HaloMode) to an instantiation.
StencilKernel stencil_kernel(ElemType type, HaloMode mode) {
  StencilKernel k = nullptr;
  with_field_type(type, "halo_stencil", [&](auto tag) {
    using T = typename decltype(tag)::type;
    switch (mode) {
      case HaloMode::kNone: k = halo_stencil_kernel<T, 0>; break;
      case HaloMode::kPull: k = halo_stencil_kernel<T, 1>; break;
      case HaloMode::kPush: k = halo_stencil_kernel<T, 2>; break;
    }
  });
  return k;
}

// Resident CTAs per SM of a stencil kernel on the current device.  One occupancy query per (kernel, device), that is
// per (type, mode, device), not per launch (per-step launches come here K times).
int occupancy_of(StencilKernel kernel) {
  static std::mutex mu;
  static std::map<std::pair<StencilKernel, int>, int> per_sm;
  int device = 0;
  HPCP_CUDA(cudaGetDevice(&device));
  std::lock_guard<std::mutex> lk(mu);
  int& n = per_sm[{kernel, device}];
  if (n == 0) HPCP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kHaloThreads, 0));
  return n;
}

struct HaloGeometry {
  StencilKernel kernel;
  uint32_t tile_bytes;
  int ctas;
};

HaloGeometry halo_geometry(size_t row_bytes, const HaloTuning& tune, HaloMode mode, int device, ElemType type) {
  HaloGeometry g;
  HPCP_REQUIRE(tune.tile_kb >= 0 && tune.tile_kb <= 1024, "halo_stencil: tile_kb in 1 .. 1024 (0 -> 16)");
  g.tile_bytes = static_cast<uint32_t>((tune.tile_kb > 0 ? tune.tile_kb : kHaloDefaultTileKb) * 1024);
  const int sms = device_sm_count(device);
  g.kernel = stencil_kernel(type, mode);
  // Co-residency: a persistent multi-step launch spins on neighbour words, so every CTA must be resident.
  const int per_sm = occupancy_of(g.kernel);
  HPCP_REQUIRE(per_sm >= 1, "halo_stencil: kernel does not fit on an SM");
  const size_t tiles = (row_bytes + g.tile_bytes - 1) / g.tile_bytes;
  const int resident = std::min(sms * std::min(per_sm, kHaloCtasPerSm), kHaloMaxCtas);  // one step word per CTA
  const int want = tune.ctas > 0 ? std::min(tune.ctas, resident) : resident;
  g.ctas = static_cast<int>(std::max<size_t>(1, std::min<size_t>(tiles, static_cast<size_t>(want))));
  HPCP_REQUIRE(g.ctas <= kHaloMaxCtas, "halo_stencil: more CTAs than flag words");
  return g;
}

}  // namespace

int halo_stencil_ctas(size_t row_elems, const HaloTuning& tune, HaloMode mode, int device, ElemType type) {
  return halo_geometry(row_elems * elem_size(type), tune, mode, device, type).ctas;
}

int launch_halo_stencil(const HaloStencilArgs& a, HaloMode mode, const HaloTuning& tune, int device,
                        cudaStream_t stream) {
  const size_t row_bytes = a.row_elems * elem_size(a.type);
  HPCP_REQUIRE(a.rows >= 1 && a.row_elems > 0 && row_bytes % 16 == 0,
               "halo_stencil: rows >= 1 and a row a positive multiple of 16 bytes");
  HPCP_REQUIRE(a.steps >= 1, "halo_stencil: steps >= 1");
  HPCP_REQUIRE(a.u[0] != nullptr && a.u[1] != nullptr, "halo_stencil: both field buffers are needed");
  const HaloGeometry g = halo_geometry(row_bytes, tune, mode, device, a.type);
  const int ctas = g.ctas;
  const size_t tiles_per_row = (row_bytes + g.tile_bytes - 1) / g.tile_bytes;
  HaloParams p{};
  for (int q = 0; q < 2; ++q) {
    p.u[q] = static_cast<float4*>(a.u[q]);
    if (mode == HaloMode::kPull) {
      HPCP_REQUIRE(a.left_u[q] != nullptr && a.right_u[q] != nullptr, "halo_stencil: pull needs the neighbours' fields");
      p.up_src[q] =
          reinterpret_cast<const float4*>(static_cast<const char*>(a.left_u[q]) + static_cast<size_t>(a.rows - 1) * row_bytes);
      p.dn_src[q] = static_cast<const float4*>(a.right_u[q]);
    } else {
      HPCP_REQUIRE(a.halo_lo[q] != nullptr && a.halo_hi[q] != nullptr, "halo_stencil: halo buffers are needed");
      p.up_src[q] = static_cast<const float4*>(a.halo_lo[q]);
      p.dn_src[q] = static_cast<const float4*>(a.halo_hi[q]);
    }
    if (mode == HaloMode::kPush) {
      HPCP_REQUIRE(a.left_halo_hi[q] != nullptr && a.right_halo_lo[q] != nullptr,
                   "halo_stencil: push needs the neighbours' halo buffers");
      p.put_first[q] = static_cast<float4*>(a.left_halo_hi[q]);
      p.put_last[q] = static_cast<float4*>(a.right_halo_lo[q]);
    }
  }
  if (mode != HaloMode::kNone) {
    HPCP_REQUIRE(a.flags_local != nullptr && a.flags_left != nullptr && a.flags_right != nullptr,
                 "halo_stencil: neighbour flag words are needed");
    HPCP_REQUIRE(a.flag_set >= 0 && a.flag_set < kHaloFlagSets, "halo_stencil: flag_set out of range");
  }
  p.rows = a.rows;
  p.cols.row_vec = row_bytes / 16;
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
  if (mode != HaloMode::kNone) {
    p.wait_lo = a.flags_local + set_words;
    p.wait_hi = a.flags_local + set_words + side_words;
    p.signal_lo = a.flags_left + set_words + side_words;  // I am the right neighbour of my left neighbour
    p.signal_hi = a.flags_right + set_words;              // and the left neighbour of my right neighbour
    p.pace = a.flags_local + set_words + 1;               // word 1 of CTA 0's sector of the wait_lo side (unused)
  }
  g.kernel<<<ctas, kHaloThreads, 0, stream>>>(p);
  HPCP_CUDA(cudaGetLastError());
  return ctas;
}

void launch_halo_init(void* u, void* halo_lo, void* halo_hi, int rows, size_t row_elems, int rank, int world,
                      cudaStream_t stream, ElemType type) {
  const int threads = 256;
  const int ctas = std::max(static_cast<int>(std::min<size_t>((row_elems + threads - 1) / threads, 132 * 8)), 1);
  with_field_type(type, "halo_init", [&](auto tag) {
    using T = typename decltype(tag)::type;
    halo_init_kernel<T><<<ctas, threads, 0, stream>>>(static_cast<T*>(u), static_cast<T*>(halo_lo),
                                                      static_cast<T*>(halo_hi), rows, row_elems, rank, world);
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_halo_verify_from_init(const void* u, int rows, size_t row_elems, int rank, int world, uint32_t steps,
                                  float alpha, float s, unsigned long long* mismatch_count, cudaStream_t stream,
                                  ElemType type) {
  HPCP_REQUIRE(rows * world <= kHaloMaxGlobalRows, "halo verify: world * rows exceeds 128 global rows");
  const int threads = 128;
  const int ctas = std::max(static_cast<int>(std::min<size_t>((row_elems + threads - 1) / threads, 132 * 16)), 1);
  with_field_type(type, "halo_verify_from_init", [&](auto tag) {
    using T = typename decltype(tag)::type;
    halo_verify_init_kernel<T><<<ctas, threads, 0, stream>>>(static_cast<const T*>(u), rows, row_elems, rank, world,
                                                             steps, alpha, s, mismatch_count);
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_halo_verify_step(const void* u_new, const void* u_old, const void* up_row, const void* dn_row, int rows,
                             size_t row_elems, float alpha, float s, unsigned long long* mismatch_count,
                             cudaStream_t stream, ElemType type) {
  const int threads = 256;
  const size_t nvec = row_elems * elem_size(type) / 16;
  const int ctas = std::max(static_cast<int>(std::min<size_t>((nvec + threads - 1) / threads, 132 * 8)), 1);
  with_field_type(type, "halo_verify_step", [&](auto tag) {
    using T = typename decltype(tag)::type;
    auto c = [](const void* q) { return static_cast<const T*>(q); };
    halo_verify_step_kernel<T><<<ctas, threads, 0, stream>>>(c(u_new), c(u_old), c(up_row), c(dn_row), rows,
                                                             row_elems, alpha, s, mismatch_count);
  });
  HPCP_CUDA(cudaGetLastError());
}

}  // namespace hpcp
