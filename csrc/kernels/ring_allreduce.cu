// Allreduce miniapp kernels (float and int).
//
// Reference pattern (aurora.mpich.miniapps/src/allreduce/mpi-sycl/allreduce-mpi-sycl.cpp:173-182):
//     Accumulate(VA,VC).wait();
//     for s in 1..P-1: { SendRecvRing(VA -> right, VB <- left); swap(VA,VB); Accumulate(VA,VC).wait(); }
// i.e. kernel -> host wait -> blocking MPI -> host wait, P-1 times: zero overlap.
//
// K-ring (this file) keeps the same data movement — every rank forwards a full
// N-element block to its right neighbour P-1 times and accumulates P blocks —
// but as ONE persistent kernel per rank: for hop t and chunk c a CTA
//   waits (acquire) on arrival word c   -> the left neighbour wrote hop t of chunk c
//   reads the chunk ONCE                -> adds it into VC and, if t < P-1,
//   stores it into the right neighbour's slot t over NVLink (peer-mapped pointer)
//   publishes (release) arrival word c  on the right neighbour.
// Accumulate, send, receive and the step barrier are fused; steps pipeline
// across the ring chunk by chunk.  By default the receive slots are (P-1) full blocks, so
// no ack channel is needed (896 MiB at P=8, N=2^25 floats — small against 180 GB of HBM3e).
// n_slots = 2 is the reference's own VA/VB double buffer (allreduce-mpi-sycl.cpp:167-168,
// 176-181): hop t lands in slot t % 2, and before a rank overwrites its neighbour's slot at
// hop t >= 2 it waits for the neighbour's per-chunk ack of hop t-1 — the flow control that a
// blocking MPI_Recv provides implicitly.  2 blocks instead of P-1 (256 MiB at P=8).
//
// The `-a` path (↔ MPI_Allreduce, :61-67) is a one-launch collective: two-shot
// over peer mappings, or NVLS (multimem.ld_reduce / multimem.st) when a
// multicast mapping exists.
#include "api.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>
#include <initializer_list>
#include <type_traits>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
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

// 16-bit floating types: two-shot accumulates them in fp32 and rounds once (two_shot_f32_kernel).
template <typename T>
constexpr bool kSum16InF32 = std::is_same<T, __nv_bfloat16>::value || std::is_same<T, __half>::value;

// The eight lanes of a 16-byte vector of T (bf16 or fp16) as fp32 partial sums: set / add widen exactly, round()
// rounds every lane once to nearest even in T (F2FP.*.F32.PACK_AB).  The fp32 adds are IEEE (no FTZ).
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
template <typename T>
struct Sum8 {
  float2 v[4];
  __device__ __forceinline__ void set(const uint4& a) {
    v[0] = Acc8<T>::widen(a.x), v[1] = Acc8<T>::widen(a.y), v[2] = Acc8<T>::widen(a.z), v[3] = Acc8<T>::widen(a.w);
  }
  __device__ __forceinline__ void add(const uint4& a) {
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = Acc8<T>::widen(w[k]);
      v[k].x = __fadd_rn(v[k].x, f.x);
      v[k].y = __fadd_rn(v[k].y, f.y);
    }
  }
  __device__ __forceinline__ uint4 round() const {
    return make_uint4(Acc8<T>::narrow(v[0].x, v[0].y), Acc8<T>::narrow(v[1].x, v[1].y),
                      Acc8<T>::narrow(v[2].x, v[2].y), Acc8<T>::narrow(v[3].x, v[3].y));
  }
};

// Element -> double for the mismatch count (the 16-bit floats convert through their exact fp32 value).
template <typename T>
__device__ __forceinline__ double to_double(T x) {
  return static_cast<double>(x);
}
__device__ __forceinline__ double to_double(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ double to_double(__half x) { return __half2float(x); }

// C++ element type -> the addition class its kernels are instantiated for.
template <typename T> struct AddClass { using type = T; };
template <> struct AddClass<unsigned int> { using type = int; };
template <> struct AddClass<unsigned long long> { using type = long long; };
template <> struct AddClass<unsigned short> { using type = short; };

// Run f(T{}) with the C++ type of `t`.
template <typename F>
void dispatch_elem(ElemType t, F&& f) {
  switch (t) {
    case ElemType::kFloat: f(float{}); break;
    case ElemType::kInt: f(int{}); break;
    case ElemType::kUInt: f(static_cast<unsigned int>(0)); break;
    case ElemType::kDouble: f(double{}); break;
    case ElemType::kLong: f(static_cast<long long>(0)); break;
    case ElemType::kULong: f(static_cast<unsigned long long>(0)); break;
    case ElemType::kShort: f(static_cast<short>(0)); break;
    case ElemType::kUShort: f(static_cast<unsigned short>(0)); break;
    case ElemType::kUChar: f(static_cast<unsigned char>(0)); break;
    case ElemType::kBFloat16: f(__nv_bfloat16{}); break;
    case ElemType::kHalf: f(__half{}); break;
  }
}
// Run f(C{}) with the addition class of `t` (eight kernel instantiations instead of eleven).
template <typename F>
void dispatch_add_class(ElemType t, F&& f) {
  dispatch_elem(t, [&](auto tag) { f(typename AddClass<decltype(tag)>::type{}); });
}

// ------------------------------------------------------------ small kernels ----
template <typename T>
__global__ void init3_kernel(T* va, T* vb, T* vc, size_t n, T a, T b, T c) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (va) va[i] = a;
    if (vb) vb[i] = b;
    if (vc) vc[i] = c;
  }
}

template <typename T>
__global__ void accumulate_kernel(const uint4* __restrict__ va, uint4* __restrict__ vc, size_t nvec,
                                  const T* va_tail, T* vc_tail, size_t tail) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride)
    vc[i] = Vec4<typename AddClass<T>::type>::add(vc[i], ptx::ld_weak_v4(va + i));
  if (blockIdx.x == 0 && threadIdx.x < tail) vc_tail[threadIdx.x] = static_cast<T>(vc_tail[threadIdx.x] + va_tail[threadIdx.x]);
}

template <typename T>
__global__ void count_mismatch_kernel(const T* __restrict__ v, size_t n, double expected,
                                      unsigned long long* count) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double d = to_double(__ldcg(v + i)) - expected;
    bad += !(d < 1e-6 && d > -1e-6);
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(count, bad);
}

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
  // kAck only (appended so that the layout the default instantiation reads is unchanged):
  uint32_t* ack_local;  // n_chunks words written by the right neighbour: "hop t of chunk c consumed"
  uint32_t* ack_left;   // peer-mapped: the left neighbour's ack words
};

// kAck = false: P-1 receive slots, hop t lands in slot t-1.  kAck = true: two slots, hop t lands in slot
// (t-1) % 2 and the sender waits for the receiver's ack of hop t-1 before it overwrites the slot at hop t+1.
template <typename T, bool kAck = false>
__global__ void __launch_bounds__(512) ring_allreduce_kernel(const __grid_constant__ RingDev a) {
  __shared__ int ok_s;
  for (int t = 0; t < a.world; ++t) {
    const uint4* src = t == 0 ? a.va : a.slots_local + static_cast<size_t>(ring_src_slot(t, kAck)) * a.nvec;
    uint4* fwd = ring_forwards(t, a.world) ? a.slots_right + static_cast<size_t>(ring_fwd_slot(t, kAck)) * a.nvec
                                           : nullptr;
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
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] = a.vc[i + k * blockDim.x];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (fwd) ptx::st_stream_v4(fwd + i + k * blockDim.x, x[k]);
          a.vc[i + k * blockDim.x] = Vec4<T>::add(acc[k], x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        const uint4 x = ptx::ld_weak_v4(src + i);
        if (fwd) ptx::st_stream_v4(fwd + i, x);
        a.vc[i] = Vec4<T>::add(a.vc[i], x);
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

template <typename T, bool kTwoSlots>
__global__ void __launch_bounds__(512) ring_pull_kernel(const __grid_constant__ RingPullDev a) {
  __shared__ int ok_s;
  for (int t = 0; t < a.world; ++t) {
    const uint4* src = t == 0   ? a.va
                       : t == 1 ? a.va_left
                                : a.slots_left + static_cast<size_t>(ring_pull_src_slot(t, kTwoSlots)) * a.nvec;
    uint4* copy = ring_pull_keeps_copy(t, a.world)
                      ? a.slots_local + static_cast<size_t>(ring_pull_copy_slot(t, kTwoSlots)) * a.nvec
                      : nullptr;
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
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] = a.vc[i + k * blockDim.x];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (copy) copy[i + k * blockDim.x] = x[k];
          a.vc[i + k * blockDim.x] = Vec4<T>::add(acc[k], x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        const uint4 x = t == 0 ? ptx::ld_weak_v4(src + i) : ptx::ld_peer_v4(src + i);
        if (copy) copy[i] = x;
        a.vc[i] = Vec4<T>::add(a.vc[i], x);
      }
      __syncthreads();  // the chunk's copy is complete (and ok_s consumed by everyone)
      // "hop t of chunk c can be read from me": VA at hop 0 (always there), the copy at hops 1 .. P-2.
      if (t + 1 < a.world && threadIdx.x == 0) publish_epoch_light(a.arrived_right + c, a.epoch_base + t + 1);
      if (kTwoSlots && ring_pull_publishes_ack(t, a.world) && threadIdx.x == 0)
        publish_epoch_light(a.ack_left + c, a.epoch_base + t);
    }
  }
}

// ------------------------------------------------- K-ring, reduce-scatter + all-gather ----
// Bandwidth-optimal ring: segment s (nvec / P vectors) of the block is reduced hop by hop on its way to rank s, then
// the finished segments travel once more round the ring.  Per (hop, chunk) a CTA waits on arrival word c, reads the
// chunk once (slot + own VA while reducing, own VC while gathering), stores it into the right neighbour's slot or VC
// and, at hop P-1, into its own VC, then publishes arrival word c on the right neighbour.  Rules: ring_order.h.
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

template <typename T>
__global__ void __launch_bounds__(512) ring_rsag_kernel(const __grid_constant__ RingRsAgDev a) {
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
          for (int k = 0; k < 4; ++k) x[k] = Vec4<T>::add(s[k], x[k]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (own) own[i + k * blockDim.x] = x[k];
          if (fwd) ptx::st_stream_v4(fwd + i + k * blockDim.x, x[k]);
        }
      }
      for (; i < end; i += blockDim.x) {
        uint4 x = ptx::ld_weak_v4(src + i);
        if (slot) x = Vec4<T>::add(ptx::ld_weak_v4(slot + i), x);
        if (own) own[i] = x;
        if (fwd) ptx::st_stream_v4(fwd + i, x);
      }
      __syncthreads();  // whole chunk stored by this CTA (and ok_s consumed by everyone)
      if (fwd && threadIdx.x == 0)
        publish_epoch_light(a.arrived_right + c, a.epoch_base + rsag_arrival(h + 1, a.phases, a.world));
    }
  }
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
// up to U*W independent NVLink loads in flight per thread.
template <typename T, int W, int U>
__global__ void __launch_bounds__(512) two_shot_kernel(const __grid_constant__ TwoShotDev a) {
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
        for (int u = 0; u < U; ++u) x[0][u] = Vec4<T>::add(x[0][u], x[q][u]);
      }
#pragma unroll
    for (int q = 0; q < W; ++q)
      if (q < a.world) {
        const int p = (a.rank + q) % a.world;
#pragma unroll
        for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[p] + base + i + u * blockDim.x, x[0][u]);
      }
  }
  size_t i = n_blocks * block_vec + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i < a.slice_vec; i += stride) {
    uint4 acc = ptx::ld_peer_v4(a.va[0] + base + i);
    for (int p = 1; p < a.world; ++p) acc = Vec4<T>::add(acc, ptx::ld_peer_v4(a.va[p] + base + i));
    for (int p = 0; p < a.world; ++p) ptx::st_stream_v4(a.vc[p] + base + i, acc);
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch,
                         a.timeout_ns, a.status);
}

// Two-shot for the 16-bit floating types: same loads, stores and barrier as two_shot_kernel, but every lane is widened
// to fp32 and the P inputs are added owner first, ((VA[s] + VA[s+1]) + ...) + VA[s+P-1] (ranks mod P), in the main
// blocks and in the tail loop alike; the sum is rounded once to T.  One rounding instead of the ring's P-1.
template <typename T, int W, int U>
__global__ void __launch_bounds__(512) two_shot_f32_kernel(const __grid_constant__ TwoShotDev a) {
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
      Sum8<T> s;
      s.set(x[0][u]);
#pragma unroll
      for (int q = 1; q < W; ++q)
        if (q < a.world) s.add(x[q][u]);
      x[0][u] = s.round();
    }
#pragma unroll
    for (int q = 0; q < W; ++q)
      if (q < a.world) {
        const int p = (a.rank + q) % a.world;
#pragma unroll
        for (int u = 0; u < U; ++u) ptx::st_stream_v4(a.vc[p] + base + i + u * blockDim.x, x[0][u]);
      }
  }
  size_t i = n_blocks * block_vec + static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i < a.slice_vec; i += stride) {
    Sum8<T> s;
    s.set(ptx::ld_peer_v4(a.va[a.rank] + base + i));
    for (int q = 1; q < a.world; ++q) s.add(ptx::ld_peer_v4(a.va[(a.rank + q) % a.world] + base + i));
    const uint4 r = s.round();
    for (int p = 0; p < a.world; ++p) ptx::st_stream_v4(a.vc[p] + base + i, r);
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch,
                         a.timeout_ns, a.status);
}

// -------------------------------------------------------------------- NVLS ----
struct NvlsDev {
  const unsigned char* va_mc;
  unsigned char* vc_mc;
  uint32_t* pads[kApiMaxRanks];
  uint32_t* ticket;
  uint32_t ticket_target;
  int rank;
  int world;
  size_t slice_vec;
  uint32_t barrier_epoch;
  uint64_t timeout_ns;
  uint32_t* status;
};

// U independent in-switch reductions in flight per thread; kMaxThreads bounds the block size (register budget).
template <typename T, int U, int kMaxThreads>
__global__ void __launch_bounds__(kMaxThreads) nvls_kernel(const __grid_constant__ NvlsDev a) {
  const size_t base = static_cast<size_t>(a.rank) * a.slice_vec;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  auto reduce_at = [&](size_t off) {
    float4 r;
    if (std::is_floating_point<T>::value) {
      r = ptx::multimem_ld_reduce_add_f32x4(a.va_mc + off);
    } else {  // int: scalar in-switch adds (no vector integer multimem.add), vector broadcast of the bits
      r.x = __int_as_float(ptx::multimem_ld_reduce_add_s32(a.va_mc + off));
      r.y = __int_as_float(ptx::multimem_ld_reduce_add_s32(a.va_mc + off + 4));
      r.z = __int_as_float(ptx::multimem_ld_reduce_add_s32(a.va_mc + off + 8));
      r.w = __int_as_float(ptx::multimem_ld_reduce_add_s32(a.va_mc + off + 12));
    }
    return r;
  };
  // Grid-stride with U (default 4) independent in-switch reductions in flight per thread.
  size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < a.slice_vec; i += U * stride) {
    float4 r[U];
#pragma unroll
    for (int k = 0; k < U; ++k) r[k] = reduce_at((base + i + k * stride) * 16);
#pragma unroll
    for (int k = 0; k < U; ++k) ptx::multimem_st_f32x4(a.vc_mc + (base + i + k * stride) * 16, r[k]);
  }
  for (; i < a.slice_vec; i += stride)
    ptx::multimem_st_f32x4(a.vc_mc + (base + i) * 16, reduce_at((base + i) * 16));
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch,
                         a.timeout_ns, a.status);
}

// Integer environment knob restricted to a list of allowed values (anything else -> the default).
int env_choice(const char* name, std::initializer_list<int> allowed, int fallback) {
  const char* e = std::getenv(name);
  if (e == nullptr) return fallback;
  const int v = std::atoi(e);
  for (int a : allowed)
    if (a == v) return v;
  return fallback;
}

int grid_for(size_t items, int threads, int cap) {
  const size_t want = (items + threads - 1) / threads;
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(want, static_cast<size_t>(cap))));
}

// Grid of a ring kernel whose CTAs own chunks round-robin.  All CTAs may spin on arrival (and ack) words, so the whole
// grid must be co-resident: clamp it with the real occupancy of the instantiation that is about to run (512 threads x
// its register count), never with a guess.  Ranks that share a GPU divide the clamp among themselves on the caller's
// side (`ctas`).
int ring_grid(const void* kernel, size_t n_chunks, int ctas, int device) {
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

}  // namespace

void launch_init3(void* va, void* vb, void* vc, size_t n, double a, double b, double c,
                  ElemType type, cudaStream_t stream) {
  const int ctas = grid_for(n, 256, 132 * 8);
  dispatch_elem(type, [&](auto tag) {
    using T = decltype(tag);
    init3_kernel<T><<<ctas, 256, 0, stream>>>(static_cast<T*>(va), static_cast<T*>(vb), static_cast<T*>(vc), n,
                                              static_cast<T>(a), static_cast<T>(b), static_cast<T>(c));
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_accumulate(const void* va, void* vc, size_t n, ElemType type, cudaStream_t stream) {
  const size_t lanes = 16 / elem_size(type);
  const size_t nvec = n / lanes, tail = n % lanes;
  const int ctas = grid_for(std::max<size_t>(nvec, 1), 512, 132 * 4);
  dispatch_elem(type, [&](auto tag) {
    using T = decltype(tag);
    accumulate_kernel<T><<<ctas, 512, 0, stream>>>(static_cast<const uint4*>(va), static_cast<uint4*>(vc), nvec,
                                                   static_cast<const T*>(va) + nvec * lanes,
                                                   static_cast<T*>(vc) + nvec * lanes, tail);
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_count_mismatch(const void* v, size_t n, double expected, ElemType type,
                           unsigned long long* count, cudaStream_t stream) {
  const int ctas = grid_for(n, 256, 132 * 8);
  dispatch_elem(type, [&](auto tag) {
    using T = decltype(tag);
    count_mismatch_kernel<T><<<ctas, 256, 0, stream>>>(static_cast<const T*>(v), n, expected, count);
  });
  HPCP_CUDA(cudaGetLastError());
}

constexpr size_t kRingDefaultChunkBytes = 128 * 1024;  // payload per arrival word

size_t ring_num_chunks(size_t n, size_t chunk_elems, size_t elem_bytes) {
  const size_t ce = chunk_elems == 0 ? kRingDefaultChunkBytes / elem_bytes : chunk_elems;
  return (n + ce - 1) / ce;
}

void launch_ring_allreduce(const RingArgs& args, ElemType type, int ctas, int device,
                           cudaStream_t stream) {
  HPCP_REQUIRE(args.world >= 1 && args.world <= kApiMaxRanks, "ring: world out of range");
  const size_t esz = elem_size(type), lanes = 16 / esz;
  HPCP_REQUIRE(args.n % lanes == 0, "ring: the block must be a multiple of 16 bytes");
  const size_t ce = args.chunk_elems == 0 ? kRingDefaultChunkBytes / esz : args.chunk_elems;
  HPCP_REQUIRE(ce % lanes == 0, "ring: a chunk must be a multiple of 16 bytes");
  RingDev d{};
  d.va = static_cast<const uint4*>(args.va);
  d.vc = static_cast<uint4*>(args.vc);
  d.slots_local = static_cast<const uint4*>(args.slots_local);
  d.slots_right = static_cast<uint4*>(args.slots_right);
  d.arrived_local = args.arrived_local;
  d.arrived_right = args.arrived_right;
  d.world = args.world;
  d.nvec = args.n / lanes;
  d.chunk_vec = ce / lanes;
  d.n_chunks = ring_num_chunks(args.n, ce, esz);
  d.epoch_base = args.epoch_base;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  const bool ack = args.n_slots == 2 && args.world > 3 && !args.pull;  // with P <= 3 no slot is ever written twice
  HPCP_REQUIRE(args.n_slots == 0 || args.n_slots == 2 || args.n_slots == args.world - 1,
               "ring: n_slots must be 0 (= world-1, no flow control) or 2 (double buffer + acks)");
  HPCP_REQUIRE(!ack || (args.ack_local != nullptr && args.ack_left != nullptr), "ring: n_slots=2 needs the ack words");
  d.ack_local = args.ack_local;
  d.ack_left = args.ack_left;
  HPCP_REQUIRE(!args.pull || args.world == 1 ||
                   (args.va_left != nullptr && (args.world == 2 || args.slots_left != nullptr)),
               "ring: the pull variant needs the left neighbour's VA and slots (peer-mapped)");
  HPCP_REQUIRE(!args.pull || args.n_slots != 2 || args.world <= 4 ||
                   (args.ack_local != nullptr && args.ack_left != nullptr),
               "ring: pull with n_slots=2 needs the ack words");
  const bool two_slots_k = args.n_slots == 2;
  const void* kernel = nullptr;
  dispatch_add_class(type, [&](auto tag) {
    using C = decltype(tag);
    if (args.pull)
      kernel = two_slots_k ? reinterpret_cast<const void*>(ring_pull_kernel<C, true>)
                           : reinterpret_cast<const void*>(ring_pull_kernel<C, false>);
    else
      kernel = two_slots_k ? reinterpret_cast<const void*>(ring_allreduce_kernel<C, true>)
                           : reinterpret_cast<const void*>(ring_allreduce_kernel<C, false>);
  });
  const int grid = ring_grid(kernel, d.n_chunks, ctas, device);
  const bool two_slots = args.n_slots == 2;  // slot index t % 2 even when no ack is ever needed (P <= 3)
  if (args.pull) {
    RingPullDev p{};
    p.va = d.va;
    p.vc = d.vc;
    p.va_left = static_cast<const uint4*>(args.va_left);
    p.slots_left = static_cast<const uint4*>(args.slots_left);
    p.slots_local = static_cast<uint4*>(args.slots_local);
    p.arrived_local = d.arrived_local;
    p.arrived_right = d.arrived_right;
    p.ack_local = args.ack_local;
    p.ack_left = args.ack_left;
    p.world = d.world;
    p.nvec = d.nvec;
    p.chunk_vec = d.chunk_vec;
    p.n_chunks = d.n_chunks;
    p.epoch_base = d.epoch_base;
    p.timeout_ns = d.timeout_ns;
    p.status = d.status;
    dispatch_add_class(type, [&](auto tag) {
      using C = decltype(tag);
      if (two_slots)
        ring_pull_kernel<C, true><<<grid, 512, 0, stream>>>(p);
      else
        ring_pull_kernel<C, false><<<grid, 512, 0, stream>>>(p);
    });
    HPCP_CUDA(cudaGetLastError());
    return;
  }
  dispatch_add_class(type, [&](auto tag) {
    using C = decltype(tag);
    if (two_slots)
      ring_allreduce_kernel<C, true><<<grid, 512, 0, stream>>>(d);
    else
      ring_allreduce_kernel<C, false><<<grid, 512, 0, stream>>>(d);
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_ring_rsag(const RingRsAgArgs& args, ElemType type, int ctas, int device, cudaStream_t stream) {
  HPCP_REQUIRE(args.world >= 1 && args.world <= kApiMaxRanks, "ring-rsag: world out of range");
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "ring-rsag: rank out of range");
  HPCP_REQUIRE(args.phases == kRsAgAllreduce || args.phases == kRsAgReduceScatter || args.phases == kRsAgAllGather,
               "ring-rsag: phases must be allreduce, reduce_scatter or all_gather");
  const size_t esz = elem_size(type), lanes = 16 / esz;
  HPCP_REQUIRE(args.n % (lanes * static_cast<size_t>(args.world)) == 0,
               "ring-rsag: every rank's segment must be a multiple of 16 bytes");
  const size_t ce = args.chunk_elems == 0 ? kRingDefaultChunkBytes / esz : args.chunk_elems;
  HPCP_REQUIRE(ce % lanes == 0, "ring-rsag: a chunk must be a multiple of 16 bytes");
  const auto va = reinterpret_cast<uintptr_t>(args.va), vc = reinterpret_cast<uintptr_t>(args.vc);
  const uintptr_t bytes = args.n * esz;
  HPCP_REQUIRE(va + bytes <= vc || vc + bytes <= va, "ring-rsag: VA and VC must not overlap (no in-place operation)");
  RingRsAgDev d{};
  d.va = static_cast<const uint4*>(args.va);
  d.vc = static_cast<uint4*>(args.vc);
  d.slots_local = static_cast<const uint4*>(args.slots_local);
  d.slots_right = static_cast<uint4*>(args.slots_right);
  d.vc_right = static_cast<uint4*>(args.vc_right);
  d.arrived_local = args.arrived_local;
  d.arrived_right = args.arrived_right;
  d.rank = args.rank;
  d.world = args.world;
  d.phases = args.phases;
  d.seg_vec = args.n / lanes / args.world;
  d.chunk_vec = ce / lanes;
  d.n_chunks = ring_num_chunks(args.n / args.world, ce, esz);
  d.epoch_base = args.epoch_base;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  dispatch_add_class(type, [&](auto tag) {
    using C = decltype(tag);
    const int grid = ring_grid(reinterpret_cast<const void*>(ring_rsag_kernel<C>), d.n_chunks, ctas, device);
    ring_rsag_kernel<C><<<grid, 512, 0, stream>>>(d);
  });
  HPCP_CUDA(cudaGetLastError());
}

int launch_allreduce_two_shot(const TwoShotArgs& args, ElemType type, int ctas, int device,
                              cudaStream_t stream) {
  HPCP_REQUIRE(args.world >= 1 && args.world <= kApiMaxRanks, "two-shot: world out of range");
  const size_t lanes = 16 / elem_size(type);
  HPCP_REQUIRE(args.n % (lanes * static_cast<size_t>(args.world)) == 0,
               "two-shot: every rank's slice must be a multiple of 16 bytes");
  TwoShotDev d{};
  for (int p = 0; p < args.world; ++p) {
    d.va[p] = static_cast<const uint4*>(args.va[p]);
    d.vc[p] = static_cast<uint4*>(args.vc[p]);
    d.pads[p] = args.pads[p];
  }
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.slice_vec = args.n / lanes / args.world;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  const int sms = device_sm_count(device);
  const int grid = grid_for(std::max<size_t>(d.slice_vec, 1), 512, ctas > 0 ? ctas : sms * 2);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
#define HPCP_TWO_SHOT(W, U)                                                \
  do {                                                                     \
    dispatch_add_class(type, [&](auto tag) {                               \
      using C = decltype(tag);                                             \
      if constexpr (kSum16InF32<C>)                                        \
        two_shot_f32_kernel<C, W, U><<<grid, 512, 0, stream>>>(d);         \
      else                                                                 \
        two_shot_kernel<C, W, U><<<grid, 512, 0, stream>>>(d);             \
    });                                                                    \
  } while (0)
  if (args.world <= 2)
    HPCP_TWO_SHOT(2, 4);
  else if (args.world <= 4)
    HPCP_TWO_SHOT(4, 4);
  else if (args.world <= 8)
    HPCP_TWO_SHOT(8, 2);
  else
    HPCP_TWO_SHOT(16, 1);
#undef HPCP_TWO_SHOT
  HPCP_CUDA(cudaGetLastError());
  return grid;
}

int launch_allreduce_nvls(const NvlsArgs& args, ElemType type, int ctas, int device,
                          cudaStream_t stream) {
  HPCP_REQUIRE(args.world >= 1 && args.world <= kApiMaxRanks, "nvls: world out of range");
  HPCP_REQUIRE(type == ElemType::kFloat || type == ElemType::kInt || type == ElemType::kUInt,
               "nvls: multimem reductions are wired for float and 32-bit integers (use two-shot for the other types)");
  HPCP_REQUIRE(args.n % (4 * static_cast<size_t>(args.world)) == 0,
               "nvls: n must be a multiple of 4*world elements");
  NvlsDev d{};
  d.va_mc = static_cast<const unsigned char*>(args.va_mc);
  d.vc_mc = static_cast<unsigned char*>(args.vc_mc);
  for (int p = 0; p < args.world; ++p) d.pads[p] = args.pads[p];
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.slice_vec = args.n / 4 / args.world;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  // HPCP_NVLS_UNROLL=4|8 (vectors in flight per thread; default 4), HPCP_NVLS_CTAS_PER_SM=k or --ctas / ctas>0 (grid).
  static const int unroll = env_choice("HPCP_NVLS_UNROLL", {4, 8}, 4);
  static const int per_sm = env_choice("HPCP_NVLS_CTAS_PER_SM", {0, 1, 2, 3, 4}, 0);
  constexpr int threads = 512;
  const int sms = device_sm_count(device);
  // Default grid: 32 CTAs.  The in-switch reduction saturates at modest request parallelism and more requesters only
  // queue in the switch.  HPCP_NVLS_CTAS_PER_SM / --ctas override.
  const int grid = grid_for(std::max<size_t>(d.slice_vec, 1), threads, ctas > 0 ? ctas : per_sm > 0 ? sms * per_sm : 32);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
#define HPCP_NVLS(U)                                                  \
  do {                                                                \
    if (type == ElemType::kFloat)                                     \
      nvls_kernel<float, U, threads><<<grid, threads, 0, stream>>>(d); \
    else                                                              \
      nvls_kernel<int, U, threads><<<grid, threads, 0, stream>>>(d);   \
  } while (0)
  if (unroll == 8)
    HPCP_NVLS(8);
  else
    HPCP_NVLS(4);
#undef HPCP_NVLS
  HPCP_CUDA(cudaGetLastError());
  return grid;
}

}  // namespace hpcp
