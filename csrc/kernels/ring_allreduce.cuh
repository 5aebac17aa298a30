// The allreduce kernels of ring_allreduce.cu (sum) and ring_allreduce_ops.cu (prod, min, max): the 16-byte lane
// policies, the device argument blocks, the kernel bodies, one __global__ template per kernel family and the table of
// kernel pointers the launchers pick from.  Everything is a template on a COMBINE POLICY -- a type with
// `static uint4 combine(const uint4& acc, const uint4& x)` that reduces every lane of one 16-byte vector.  The sum is
// the policy SumOp<C>; it differs from the others in two template arguments only: its rings accumulate into VC where
// the others overwrite it at hop 0 (kOverwrite), and its two-shot tail combines rank 0 first (kOwnerFirstTail).
// The argument blocks' layouts are part of the fingerprinted instruction streams (docs/sass/VALIDATED.sha256).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>
#include <utility>

#include "../common/cuda_check.h"
#include "../common/dtype_traits.h"
#include "../common/signal.cuh"
#include "api.h"
#include "ring_order.h"

namespace hpcp {

namespace {

template <typename T>
struct Vec4;
template <>
struct Vec4<float> {
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    return make_uint4(__float_as_uint(__uint_as_float(a.x) + __uint_as_float(b.x)),
                      __float_as_uint(__uint_as_float(a.y) + __uint_as_float(b.y)),
                      __float_as_uint(__uint_as_float(a.z) + __uint_as_float(b.z)),
                      __float_as_uint(__uint_as_float(a.w) + __uint_as_float(b.w)));
  }
};
template <>
struct Vec4<int> {
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    return make_uint4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
};
template <>
struct Vec4<double> {  // two f64 lanes per 16 bytes
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    const double lo = __hiloint2double(static_cast<int>(a.y), static_cast<int>(a.x)) +
                      __hiloint2double(static_cast<int>(b.y), static_cast<int>(b.x));
    const double hi = __hiloint2double(static_cast<int>(a.w), static_cast<int>(a.z)) +
                      __hiloint2double(static_cast<int>(b.w), static_cast<int>(b.z));
    return make_uint4(static_cast<uint32_t>(__double2loint(lo)), static_cast<uint32_t>(__double2hiint(lo)),
                      static_cast<uint32_t>(__double2loint(hi)), static_cast<uint32_t>(__double2hiint(hi)));
  }
};
template <>
struct Vec4<long long> {  // two 64-bit lanes (signed and unsigned share the add)
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    const unsigned long long lo = ((static_cast<unsigned long long>(a.y) << 32) | a.x) +
                                  ((static_cast<unsigned long long>(b.y) << 32) | b.x);
    const unsigned long long hi = ((static_cast<unsigned long long>(a.w) << 32) | a.z) +
                                  ((static_cast<unsigned long long>(b.w) << 32) | b.z);
    return make_uint4(static_cast<uint32_t>(lo), static_cast<uint32_t>(lo >> 32), static_cast<uint32_t>(hi),
                      static_cast<uint32_t>(hi >> 32));
  }
};
template <>
struct Vec4<short> {  // eight 16-bit lanes: per-halfword SIMD add (wraps like the scalar add)
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    return make_uint4(__vadd2(a.x, b.x), __vadd2(a.y, b.y), __vadd2(a.z, b.z), __vadd2(a.w, b.w));
  }
};
template <>
struct Vec4<unsigned char> {  // sixteen 8-bit lanes
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    return make_uint4(__vadd4(a.x, b.x), __vadd4(a.y, b.y), __vadd4(a.z, b.z), __vadd4(a.w, b.w));
  }
};
// Eight 16-bit floating lanes, two per 32-bit word (H2 = __nv_bfloat162 / __half2): every lane is ONE add rounded to
// nearest even in the 16-bit format, subnormal results kept (HFMA2.BF16_V2 a, 1, b / HFMA2 without .FTZ).
template <typename H2>
struct Vec4Pairs {
  static __device__ __forceinline__ uint32_t add2(uint32_t a, uint32_t b) {
    const H2 s = __hadd2_rn(*reinterpret_cast<const H2*>(&a), *reinterpret_cast<const H2*>(&b));
    return *reinterpret_cast<const uint32_t*>(&s);
  }
  static __device__ __forceinline__ uint4 add(const uint4& a, const uint4& b) {
    return make_uint4(add2(a.x, b.x), add2(a.y, b.y), add2(a.z, b.z), add2(a.w, b.w));
  }
};
template <>
struct Vec4<__nv_bfloat16> : Vec4Pairs<__nv_bfloat162> {};
template <>
struct Vec4<__half> : Vec4Pairs<__half2> {};

// The sum as a combine policy.
template <typename T>
struct SumOp {
  static __device__ __forceinline__ uint4 combine(const uint4& acc, const uint4& x) { return Vec4<T>::add(acc, x); }
};

// The eight lanes of a 16-byte vector of T (bf16 or fp16) as fp32 partials: set / combine widen exactly, round()
// rounds every lane once to nearest even in T (F2FP.*.F32.PACK_AB).  F is the fp32 operation (IEEE, no FTZ).
template <typename T>
struct Acc8;
template <>
struct Acc8<__nv_bfloat16> {
  static __device__ __forceinline__ float2 widen(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
  }
  static __device__ __forceinline__ uint32_t narrow(float lo, float hi) {
    const __nv_bfloat162 r = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&r);
  }
};
template <>
struct Acc8<__half> {
  static __device__ __forceinline__ float2 widen(uint32_t u) {
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
  }
  static __device__ __forceinline__ uint32_t narrow(float lo, float hi) {
    const __half2 r = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&r);
  }
};
struct AddF32 {
  static __device__ __forceinline__ float apply(float a, float b) { return __fadd_rn(a, b); }
};
template <typename T, class F>
struct Wide8 {
  float2 v[4];
  __device__ __forceinline__ void set(const uint4& a) {
    v[0] = Acc8<T>::widen(a.x), v[1] = Acc8<T>::widen(a.y), v[2] = Acc8<T>::widen(a.z), v[3] = Acc8<T>::widen(a.w);
  }
  __device__ __forceinline__ void add(const uint4& a) {
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = Acc8<T>::widen(w[k]);
      v[k].x = F::apply(v[k].x, f.x);
      v[k].y = F::apply(v[k].y, f.y);
    }
  }
  __device__ __forceinline__ uint4 round() const {
    return make_uint4(Acc8<T>::narrow(v[0].x, v[0].y), Acc8<T>::narrow(v[1].x, v[1].y),
                      Acc8<T>::narrow(v[2].x, v[2].y), Acc8<T>::narrow(v[3].x, v[3].y));
  }
};
template <typename T>
using Sum8 = Wide8<T, AddF32>;

// ------------------------------------------------------------------ K-ring ----
struct RingDev {
  const uint4* va;
  uint4* vc;
  const uint4* slots_local;
  uint4* slots_right;
  uint32_t* arrived_local;
  uint32_t* arrived_right;
  int world;
  size_t nvec;        // vectors per block
  size_t chunk_vec;   // vectors per chunk
  size_t n_chunks;
  uint32_t epoch_base;
  uint64_t timeout_ns;
  uint32_t* status;
  // kAck only:
  uint32_t* ack_local;  // n_chunks words written by the right neighbour: "hop t of chunk c consumed"
  uint32_t* ack_left;   // peer-mapped: the left neighbour's ack words
};

// kAck = false: P-1 receive slots, hop t lands in slot t-1.  kAck = true: two slots, hop t lands in slot
// (t-1) % 2 and the sender waits for the receiver's ack of hop t-1 before it overwrites the slot at hop t+1.
// kOverwrite: hop 0 stores VA into VC without reading VC (every op but the sum); otherwise VC accumulates every hop.
template <class Op, bool kAck, bool kOverwrite>
__device__ __forceinline__ void ring_push_body(const RingDev& a) {
  __shared__ int ok_s;
  for (int t = 0; t < a.world; ++t) {
    const uint4* src = t == 0 ? a.va : a.slots_local + static_cast<size_t>(ring_src_slot(t, kAck)) * a.nvec;
    uint4* fwd = ring_forwards(t, a.world) ? a.slots_right + static_cast<size_t>(ring_fwd_slot(t, kAck)) * a.nvec
                                           : nullptr;
    const bool first = kOverwrite && t == 0;
    for (size_t c = blockIdx.x; c < a.n_chunks; c += gridDim.x) {
      if (t > 0) {
        if (threadIdx.x == 0)
          ok_s = wait_epoch(a.arrived_local + c, a.epoch_base + t, a.timeout_ns, a.status) ? 1 : 0;
        __syncthreads();
        if (!ok_s) return;  // peer hung: status word set, drain
      }
      if (kAck && ring_waits_for_ack(t, a.world)) {
        // My hop-t forward overwrites what the right neighbour received at hop t-2 and reads at ITS hop t-1.
        if (threadIdx.x == 0)
          ok_s = wait_epoch(a.ack_local + c, a.epoch_base + t - 1, a.timeout_ns, a.status) ? 1 : 0;
        __syncthreads();
        if (!ok_s) return;
      }
      const size_t begin = c * a.chunk_vec;
      const size_t end = begin + a.chunk_vec < a.nvec ? begin + a.chunk_vec : a.nvec;
      size_t i = begin + threadIdx.x;
      for (; i + 3 * blockDim.x < end; i += 4 * blockDim.x) {
        uint4 x[4], acc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = ptx::ld_weak_v4(src + i + k * blockDim.x);
        if (!first) {
#pragma unroll
          for (int k = 0; k < 4; ++k) acc[k] = a.vc[i + k * blockDim.x];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (fwd) ptx::st_stream_v4(fwd + i + k * blockDim.x, x[k]);
          a.vc[i + k * blockDim.x] = first ? x[k] : Op::combine(acc[k], x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        const uint4 x = ptx::ld_weak_v4(src + i);
        if (fwd) ptx::st_stream_v4(fwd + i, x);
        a.vc[i] = first ? x : Op::combine(a.vc[i], x);
      }
      __syncthreads();  // whole chunk stored by this CTA (and ok_s consumed by everyone)
      if (fwd && threadIdx.x == 0) publish_epoch_light(a.arrived_right + c, a.epoch_base + t + 1);
      // The slot chunk I have just read may be overwritten: tell the left neighbour (it only looks at hops
      // 1 .. P-3, the ones followed by another write into the same slot).
      if (kAck && ring_publishes_ack(t, a.world) && threadIdx.x == 0)
        publish_epoch_light(a.ack_left + c, a.epoch_base + t);
    }
  }
}

template <class Op, bool kAck, bool kOverwrite>
__global__ void __launch_bounds__(512) ring_push_kernel(const __grid_constant__ RingDev a) {
  ring_push_body<Op, kAck, kOverwrite>(a);
}

// ------------------------------------------------------------ K-ring, pull variant ----
// Same data movement (every rank receives P-1 full blocks and accumulates P), but the bytes cross NVLink as LOADS
// issued by the receiver instead of stores issued by the sender (which initiative moves more bytes per second over
// the link is a measurement, not an expectation).  Per (hop, chunk):
//   wait (acquire) arrival word c  -> the left neighbour holds hop t-1 of chunk c (its VA for t = 1, else a slot)
//   load the chunk from the LEFT neighbour's memory, add it into VC, keep a local copy for the right neighbour
//   publish (release) arrival word c on the RIGHT neighbour: "hop t of chunk c can be read from me".
struct RingPullDev {
  const uint4* va;
  uint4* vc;
  const uint4* va_left;      // peer-mapped: the left neighbour's VA
  const uint4* slots_left;   // peer-mapped: the left neighbour's local copies
  uint4* slots_local;        // my copies, read by the right neighbour
  uint32_t* arrived_local;
  uint32_t* arrived_right;
  uint32_t* ack_local;       // two slots: written by the right neighbour ("hop t of chunk c read")
  uint32_t* ack_left;
  int world;
  size_t nvec, chunk_vec, n_chunks;
  uint32_t epoch_base;
  uint64_t timeout_ns;
  uint32_t* status;
};

template <class Op, bool kTwoSlots, bool kOverwrite>
__device__ __forceinline__ void ring_pull_body(const RingPullDev& a) {
  __shared__ int ok_s;
  for (int t = 0; t < a.world; ++t) {
    const uint4* src = t == 0   ? a.va
                       : t == 1 ? a.va_left
                                : a.slots_left + static_cast<size_t>(ring_pull_src_slot(t, kTwoSlots)) * a.nvec;
    uint4* copy = ring_pull_keeps_copy(t, a.world)
                      ? a.slots_local + static_cast<size_t>(ring_pull_copy_slot(t, kTwoSlots)) * a.nvec
                      : nullptr;
    const bool first = kOverwrite && t == 0;
    for (size_t c = blockIdx.x; c < a.n_chunks; c += gridDim.x) {
      if (t > 0) {
        if (threadIdx.x == 0)
          ok_s = wait_epoch(a.arrived_local + c, a.epoch_base + t, a.timeout_ns, a.status) ? 1 : 0;
        __syncthreads();
        if (!ok_s) return;
      }
      if (kTwoSlots && ring_pull_waits_for_ack(t, a.world)) {
        if (threadIdx.x == 0)
          ok_s = wait_epoch(a.ack_local + c, a.epoch_base + t - 1, a.timeout_ns, a.status) ? 1 : 0;
        __syncthreads();
        if (!ok_s) return;
      }
      const size_t begin = c * a.chunk_vec;
      const size_t end = begin + a.chunk_vec < a.nvec ? begin + a.chunk_vec : a.nvec;
      size_t i = begin + threadIdx.x;
      for (; i + 3 * blockDim.x < end; i += 4 * blockDim.x) {
        uint4 x[4], acc[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          x[k] = t == 0 ? ptx::ld_weak_v4(src + i + k * blockDim.x) : ptx::ld_peer_v4(src + i + k * blockDim.x);
        if (!first) {
#pragma unroll
          for (int k = 0; k < 4; ++k) acc[k] = a.vc[i + k * blockDim.x];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (copy) copy[i + k * blockDim.x] = x[k];
          a.vc[i + k * blockDim.x] = first ? x[k] : Op::combine(acc[k], x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        const uint4 x = t == 0 ? ptx::ld_weak_v4(src + i) : ptx::ld_peer_v4(src + i);
        if (copy) copy[i] = x;
        a.vc[i] = first ? x : Op::combine(a.vc[i], x);
      }
      __syncthreads();  // the chunk's copy is complete (and ok_s consumed by everyone)
      // "hop t of chunk c can be read from me": VA at hop 0 (always there), the copy at hops 1 .. P-2.
      if (t + 1 < a.world && threadIdx.x == 0) publish_epoch_light(a.arrived_right + c, a.epoch_base + t + 1);
      if (kTwoSlots && ring_pull_publishes_ack(t, a.world) && threadIdx.x == 0)
        publish_epoch_light(a.ack_left + c, a.epoch_base + t);
    }
  }
}

template <class Op, bool kTwoSlots, bool kOverwrite>
__global__ void __launch_bounds__(512) ring_pull_kernel(const __grid_constant__ RingPullDev a) {
  ring_pull_body<Op, kTwoSlots, kOverwrite>(a);
}

// ------------------------------------------------- K-ring, reduce-scatter + all-gather ----
// Bandwidth-optimal ring: segment s (nvec / P vectors) of the block is reduced hop by hop on its way to rank s, then
// the finished segments travel once more round the ring.  Per (hop, chunk) a CTA waits on arrival word c, reads the
// chunk once (slot + own VA while reducing, own VC while gathering), stores it into the right neighbour's slot or VC
// and, at hop P-1, into its own VC, then publishes arrival word c on the right neighbour.  Rules: ring_order.h.
// VC is only ever written before it is read, so the sum and the ops share the body as it is.
struct RingRsAgDev {
  const uint4* va;
  uint4* vc;
  const uint4* slots_local;
  uint4* slots_right;
  uint4* vc_right;
  uint32_t* arrived_local;
  uint32_t* arrived_right;
  int rank;
  int world;
  int phases;
  size_t seg_vec;     // vectors per segment
  size_t chunk_vec;   // vectors per chunk
  size_t n_chunks;    // chunks per segment
  uint32_t epoch_base;
  uint64_t timeout_ns;
  uint32_t* status;
};

template <class Op>
__device__ __forceinline__ void ring_rsag_body(const RingRsAgDev& a) {
  __shared__ int ok_s;
  const int last = rsag_last_hop(a.phases, a.world);
  for (int h = rsag_first_hop(a.phases, a.world); h <= last; ++h) {
    const size_t seg = static_cast<size_t>(rsag_segment(h, a.rank, a.world)) * a.seg_vec;
    const uint4* src = (rsag_reads_vc(h, a.world) ? a.vc : a.va) + seg;
    const int rs = rsag_src_slot(h, a.phases, a.world);
    const uint4* slot = rs >= 0 ? a.slots_local + static_cast<size_t>(rs) * a.seg_vec : nullptr;
    uint4* own = rsag_writes_own_vc(h, a.world) ? a.vc + seg : nullptr;
    const int fs = rsag_fwd_slot(h, a.world);
    uint4* fwd = !rsag_forwards(h, a.phases, a.world) ? nullptr
                 : fs >= 0                             ? a.slots_right + static_cast<size_t>(fs) * a.seg_vec
                                                       : a.vc_right + seg;
    const bool waits = rsag_waits(h, a.phases, a.world);
    const uint32_t want = a.epoch_base + rsag_arrival(h, a.phases, a.world);
    for (size_t c = blockIdx.x; c < a.n_chunks; c += gridDim.x) {
      if (waits) {
        if (threadIdx.x == 0) ok_s = wait_epoch(a.arrived_local + c, want, a.timeout_ns, a.status) ? 1 : 0;
        __syncthreads();
        if (!ok_s) return;  // peer hung: status word set, drain
      }
      const size_t begin = c * a.chunk_vec;
      const size_t end = begin + a.chunk_vec < a.seg_vec ? begin + a.chunk_vec : a.seg_vec;
      size_t i = (own || fwd) ? begin + threadIdx.x : end;  // the last hop of a gather only waits
      for (; i + 3 * blockDim.x < end; i += 4 * blockDim.x) {
        uint4 x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = ptx::ld_weak_v4(src + i + k * blockDim.x);
        if (slot) {
          uint4 s[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) s[k] = ptx::ld_weak_v4(slot + i + k * blockDim.x);
#pragma unroll
          for (int k = 0; k < 4; ++k) x[k] = Op::combine(s[k], x[k]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (own) own[i + k * blockDim.x] = x[k];
          if (fwd) ptx::st_stream_v4(fwd + i + k * blockDim.x, x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        uint4 x = ptx::ld_weak_v4(src + i);
        if (slot) x = Op::combine(ptx::ld_weak_v4(slot + i), x);
        if (own) own[i] = x;
        if (fwd) ptx::st_stream_v4(fwd + i, x);
      }
      __syncthreads();  // whole chunk stored by this CTA (and ok_s consumed by everyone)
      if (fwd && threadIdx.x == 0)
        publish_epoch_light(a.arrived_right + c, a.epoch_base + rsag_arrival(h + 1, a.phases, a.world));
    }
  }
}

template <class Op>
__global__ void __launch_bounds__(512) ring_rsag_kernel(const __grid_constant__ RingRsAgDev a) {
  ring_rsag_body<Op>(a);
}

// ---------------------------------------------------------------- two-shot ----
struct TwoShotDev {
  const uint4* va[kApiMaxRanks];
  uint4* vc[kApiMaxRanks];
  uint32_t* pads[kApiMaxRanks];
  uint32_t* ticket;
  uint32_t ticket_target;
  int rank;
  int world;
  size_t slice_vec;  // vectors per rank slice
  uint32_t barrier_epoch;
  uint64_t timeout_ns;
  uint32_t* status;
};

// After the whole grid finished its stores, the last CTA runs the cross-GPU
// barrier: kernel completion then implies every peer's slice landed in my VC.
__device__ __forceinline__ void grid_then_node_barrier(uint32_t* ticket, uint32_t ticket_target,
                                                       uint32_t* const* pads, int rank, int world,
                                                       uint32_t epoch, uint64_t timeout_ns,
                                                       uint32_t* status) {
  __shared__ int last_s;
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::fence_acq_rel_sys();
    const uint32_t t = ptx::atom_acq_rel_gpu_add(ticket, 1u);
    last_s = (t + 1u == ticket_target) ? 1 : 0;
    if (last_s) ptx::fence_acq_rel_sys();
  }
  __syncthreads();
  if (!last_s) return;
  if (static_cast<int>(threadIdx.x) < world) {
    ptx::st_release_sys(pads[threadIdx.x] + kPadBarrier + rank, epoch);
    wait_epoch(pads[rank] + kPadBarrier + threadIdx.x, epoch, timeout_ns, status);
  }
}

// W = compile-time bound on the world size (register arrays), U = vectors per thread per trip:
// up to U*W independent NVLink loads in flight per thread.  The main blocks combine owner first,
// ((VA[s] o VA[s+1]) o ...); the tail loop does too with kOwnerFirstTail, else it goes rank 0 first.
// kOwnerFirstTail is false for the sum only.  Its tail adding rank 0 first, unlike its main blocks, is part of the
// sum's results (a floating sum's last bits depend on the order) and of its fingerprinted instructions.
// kScatter: the stand-alone reduce-scatter.  va[p] is rank p's send buffer and vc[rank] my receive buffer of ONE
// segment: the result of segment `rank` is stored there only, at offset 0 (kOwnerFirstTail is true).
template <class Op, int W, int U, bool kOwnerFirstTail, bool kScatter = false>
__device__ __forceinline__ void two_shot_body(const TwoShotDev& a) {
  const size_t base = static_cast<size_t>(a.rank) * a.slice_vec;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t block_vec = static_cast<size_t>(blockDim.x) * U;
  const size_t n_blocks = a.slice_vec / block_vec;
  for (size_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const size_t i = blk * block_vec + threadIdx.x;  // CTA-contiguous block of U * blockDim vectors
    uint4 x[W][U];
#pragma unroll
    for (int q = 0; q < W; ++q)
      if (q < a.world) {
        const int p = (a.rank + q) % a.world;  // start at self, then the neighbours: spreads load
#pragma unroll
        for (int u = 0; u < U; ++u) x[q][u] = ptx::ld_peer_v4(a.va[p] + base + i + u * blockDim.x);
      }
#pragma unroll
    for (int q = 1; q < W; ++q)
      if (q < a.world) {
#pragma unroll
        for (int u = 0; u < U; ++u) x[0][u] = Op::combine(x[0][u], x[q][u]);
      }
    if constexpr (kScatter) {
#pragma unroll
      for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[a.rank] + i + u * blockDim.x, x[0][u]);
    } else {
#pragma unroll
      for (int q = 0; q < W; ++q)
        if (q < a.world) {
          const int p = (a.rank + q) % a.world;
#pragma unroll
          for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[p] + base + i + u * blockDim.x, x[0][u]);
        }
    }
  }
  size_t i = n_blocks * block_vec + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i < a.slice_vec; i += stride) {
    if (kOwnerFirstTail) {
      uint4 acc = ptx::ld_peer_v4(a.va[a.rank] + base + i);
      for (int q = 1; q < a.world; ++q) acc = Op::combine(acc, ptx::ld_peer_v4(a.va[(a.rank + q) % a.world] + base + i));
      if constexpr (kScatter)
        ptx::st_stream_v4(a.vc[a.rank] + i, acc);
      else
        for (int p = 0; p < a.world; ++p) ptx::st_stream_v4(a.vc[p] + base + i, acc);
    } else {
      uint4 acc = ptx::ld_peer_v4(a.va[0] + base + i);
      for (int p = 1; p < a.world; ++p) acc = Op::combine(acc, ptx::ld_peer_v4(a.va[p] + base + i));
      for (int p = 0; p < a.world; ++p) ptx::st_stream_v4(a.vc[p] + base + i, acc);
    }
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch,
                         a.timeout_ns, a.status);
}

template <class Op, int W, int U, bool kOwnerFirstTail>
__global__ void __launch_bounds__(512) two_shot_kernel(const __grid_constant__ TwoShotDev a) {
  two_shot_body<Op, W, U, kOwnerFirstTail>(a);
}

// The stand-alone reduce-scatter: two-shot's loads and combine order (owner first, the tail too), one store.
template <class Op, int W, int U>
__global__ void __launch_bounds__(512) reduce_scatter_kernel(const __grid_constant__ TwoShotDev a) {
  two_shot_body<Op, W, U, true, true>(a);
}

// Two-shot for the 16-bit floating types: same loads, stores and barrier as two_shot_body, but every lane is widened
// to fp32 (the accumulator A, a Wide8) and the P inputs are combined owner first, ((VA[s] o VA[s+1]) o ...) o
// VA[s+P-1] (ranks mod P), in the main blocks and in the tail loop alike; the result is rounded once to T.
// kScatter as in two_shot_body.
template <class A, int W, int U, bool kScatter = false>
__device__ __forceinline__ void two_shot_f32_body(const TwoShotDev& a) {
  const size_t base = static_cast<size_t>(a.rank) * a.slice_vec;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t block_vec = static_cast<size_t>(blockDim.x) * U;
  const size_t n_blocks = a.slice_vec / block_vec;
  for (size_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const size_t i = blk * block_vec + threadIdx.x;
    uint4 x[W][U];
#pragma unroll
    for (int q = 0; q < W; ++q)
      if (q < a.world) {
        const int p = (a.rank + q) % a.world;  // owner first: the summation order
#pragma unroll
        for (int u = 0; u < U; ++u) x[q][u] = ptx::ld_peer_v4(a.va[p] + base + i + u * blockDim.x);
      }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      A s;
      s.set(x[0][u]);
#pragma unroll
      for (int q = 1; q < W; ++q)
        if (q < a.world) s.add(x[q][u]);
      x[0][u] = s.round();
    }
    if constexpr (kScatter) {
#pragma unroll
      for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[a.rank] + i + u * blockDim.x, x[0][u]);
    } else {
#pragma unroll
      for (int q = 0; q < W; ++q)
        if (q < a.world) {
          const int p = (a.rank + q) % a.world;
#pragma unroll
          for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[p] + base + i + u * blockDim.x, x[0][u]);
        }
    }
  }
  size_t i = n_blocks * block_vec + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i < a.slice_vec; i += stride) {
    A s;
    s.set(ptx::ld_peer_v4(a.va[a.rank] + base + i));
    for (int q = 1; q < a.world; ++q) s.add(ptx::ld_peer_v4(a.va[(a.rank + q) % a.world] + base + i));
    const uint4 r = s.round();
    if constexpr (kScatter)
      ptx::st_stream_v4(a.vc[a.rank] + i, r);
    else
      for (int p = 0; p < a.world; ++p) ptx::st_stream_v4(a.vc[p] + base + i, r);
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch,
                         a.timeout_ns, a.status);
}

template <class Acc, int W, int U>
__global__ void __launch_bounds__(512) two_shot_f32_kernel(const __grid_constant__ TwoShotDev a) {
  two_shot_f32_body<Acc, W, U>(a);
}

template <class Acc, int W, int U>
__global__ void __launch_bounds__(512) reduce_scatter_f32_kernel(const __grid_constant__ TwoShotDev a) {
  two_shot_f32_body<Acc, W, U, true>(a);
}

// The combine policies two-shot runs through two_shot_f32_kernel, and the accumulator (a Wide8) each one uses: the sum
// of the 16-bit floating types here, their product in ring_allreduce_ops.cu.
template <class Op>
struct TwoShotInF32 : std::false_type {};
template <typename T>
struct TwoShotInF32<SumOp<T>> : std::integral_constant<bool, kSum16InF32<T>> {
  using acc = Sum8<T>;
};

// ------------------------------------------------------------------- grids ----
inline int grid_for(size_t items, int threads, int cap) {
  const size_t want = (items + threads - 1) / threads;
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(want, static_cast<size_t>(cap))));
}

// Grid of a ring kernel whose CTAs own chunks round-robin.  All CTAs may spin on arrival (and ack) words, so the whole
// grid must be co-resident: clamp it with the real occupancy of the instantiation that is about to run (512 threads x
// its register count), never with a guess.  Ranks that share a GPU divide the clamp among themselves on the caller's
// side (`ctas`).
inline int ring_grid(const void* kernel, size_t n_chunks, int ctas, int device) {
  int per_sm = 0;
  HPCP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 512, 0));
  HPCP_REQUIRE(per_sm >= 1, "ring: the kernel does not fit on an SM");
  const int sms = device_sm_count(device);
  int grid = ctas > 0 ? ctas : sms * std::min(per_sm, 2);
  grid = std::min(grid, sms * per_sm);
  grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(grid), std::max<size_t>(n_chunks, 1)));
  if (ctas <= 0 && n_chunks > static_cast<size_t>(grid)) {
    // Chunks are dealt round-robin: pick the grid in [3/4 cap, cap] that wastes the least
    // (every CTA should own the same number of chunks, or the slowest CTA paces the ring).
    int best = grid;
    size_t best_waste = ~size_t{0};
    for (int g = grid; g >= grid * 3 / 4 && g >= 1; --g) {
      const size_t rounds = (n_chunks + g - 1) / g;
      const size_t waste = rounds * g - n_chunks;
      // compare wasted chunk-slots relative to useful parallelism
      if (waste * best < best_waste * g || best_waste == ~size_t{0}) {
        best_waste = waste;
        best = g;
      }
      if (waste == 0) break;
    }
    grid = best;
  }
  return grid;
}

constexpr size_t kRingDefaultChunkBytes = 128 * 1024;  // payload per arrival word

}  // namespace

// --------------------------------------------------------- kernel selection ----
// Two-shot's <W, U> by world size: the first row with world <= W runs (the last one takes the rest).
struct TwoShotShape {
  int w, u;
};
constexpr TwoShotShape kTwoShotShapes[] = {{2, 4}, {4, 4}, {8, 2}, {16, 1}};
constexpr int kTwoShotShapeCount = sizeof(kTwoShotShapes) / sizeof(kTwoShotShapes[0]);
inline int two_shot_shape(int world) {
  int i = 0;
  while (i + 1 < kTwoShotShapeCount && world > kTwoShotShapes[i].w) ++i;
  return i;
}

// The kernels of one (element type, op), every one launched with 512 threads and its family's argument block.
struct AllreduceKernels {
  const void* ring[2][2];                    // [pull][two slots]: RingDev (push) or RingPullDev (pull)
  const void* rsag;                          // RingRsAgDev
  const void* two_shot[kTwoShotShapeCount];  // [two_shot_shape(world)]: TwoShotDev
  const void* reduce_scatter[kTwoShotShapeCount];  // [two_shot_shape(world)]: TwoShotDev, two_shot_body's kScatter
};

namespace {

template <class K>
const void* kernel_ptr(K* kernel) {
  return reinterpret_cast<const void*>(kernel);
}

template <class Op, bool kOwnerFirstTail, int I>
const void* two_shot_kernel_of() {
  constexpr int W = kTwoShotShapes[I].w, U = kTwoShotShapes[I].u;
  if constexpr (TwoShotInF32<Op>::value)
    return kernel_ptr(two_shot_f32_kernel<typename TwoShotInF32<Op>::acc, W, U>);
  else
    return kernel_ptr(two_shot_kernel<Op, W, U, kOwnerFirstTail>);
}

template <class Op, int I>
const void* reduce_scatter_kernel_of() {
  constexpr int W = kTwoShotShapes[I].w, U = kTwoShotShapes[I].u;
  if constexpr (TwoShotInF32<Op>::value)
    return kernel_ptr(reduce_scatter_f32_kernel<typename TwoShotInF32<Op>::acc, W, U>);
  else
    return kernel_ptr(reduce_scatter_kernel<Op, W, U>);
}

template <class Op, bool kOverwrite, bool kOwnerFirstTail, int... I>
AllreduceKernels allreduce_kernels_of(std::integer_sequence<int, I...>) {
  return {{{kernel_ptr(ring_push_kernel<Op, false, kOverwrite>), kernel_ptr(ring_push_kernel<Op, true, kOverwrite>)},
           {kernel_ptr(ring_pull_kernel<Op, false, kOverwrite>), kernel_ptr(ring_pull_kernel<Op, true, kOverwrite>)}},
          kernel_ptr(ring_rsag_kernel<Op>),
          {two_shot_kernel_of<Op, kOwnerFirstTail, I>()...},
          {reduce_scatter_kernel_of<Op, I>()...}};
}
// Every kernel of the combine policy Op.
template <class Op, bool kOverwrite, bool kOwnerFirstTail>
AllreduceKernels allreduce_kernels_of() {
  return allreduce_kernels_of<Op, kOverwrite, kOwnerFirstTail>(std::make_integer_sequence<int, kTwoShotShapeCount>{});
}

// One launch of 512 threads per CTA; `args` are the kernel's parameters, with exactly their types.
template <class... Args>
void launch_512(const void* kernel, int grid, cudaStream_t stream, Args... args) {
  void* params[] = {&args...};
  HPCP_CUDA(cudaLaunchKernel(kernel, dim3(grid), dim3(512), params, 0, stream));
}

}  // namespace

// The prod / min / max kernels (ring_allreduce_ops.cu) for the launchers of ring_allreduce.cu; `op` is not kSum.
AllreduceKernels op_allreduce_kernels(ElemType type, ReduceOp op);
// VC = op(VC, VA), parameters (const uint4* va, uint4* vc, size_t nvec, const unsigned char* va_tail,
// unsigned char* vc_tail, size_t tail_bytes).
const void* op_combine_kernel(ElemType type, ReduceOp op);

}  // namespace hpcp
