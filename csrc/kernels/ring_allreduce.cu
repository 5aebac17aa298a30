// Allreduce miniapp: the launchers of every algorithm, the sum's instantiations of the kernel templates of
// ring_allreduce.cuh (prod, min and max are instantiated in ring_allreduce_ops.cu), the NVLS kernel and the small
// init / accumulate / verify kernels.  A launcher validates, fills the device argument block, takes the kernel of
// (type, op) from allreduce_kernels() and launches it: the sum goes the same way as every other op.
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
#include "ring_allreduce.cuh"

#include <cstdlib>
#include <cstring>
#include <initializer_list>

namespace hpcp {

namespace {

// Element -> double for the mismatch count (the 16-bit floats convert through their exact fp32 value).
template <typename T>
__device__ __forceinline__ double to_double(T x) {
  return static_cast<double>(x);
}
__device__ __forceinline__ double to_double(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ double to_double(__half x) { return __half2float(x); }

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

// Pair types: W is the pair's bytes as one 8- or 16-byte word (uint2 / uint4), padding included.
template <typename W>
__global__ void fill_pair_kernel(W* v, size_t n, W pair) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) v[i] = pair;
}
__device__ __forceinline__ bool same_bits(uint2 a, uint2 b) { return a.x == b.x && a.y == b.y; }
__device__ __forceinline__ bool same_bits(uint4 a, uint4 b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }
template <typename W>
__global__ void count_pair_mismatch_kernel(const W* __restrict__ v, size_t n, W pair, unsigned long long* count) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    bad += !same_bits(__ldcg(v + i), pair);
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(count, bad);
}
// f(W{}, pair bits) for the pair (value, index) of `type`, padding zero.
template <typename F>
void with_pair_bits(ElemType type, double value, int index, F&& f) {
  dispatch_pair(type, [&](auto tag) {
    using P = decltype(tag);
    using W = std::conditional_t<sizeof(P) == 16, uint4, uint2>;
    P p;
    std::memset(static_cast<void*>(&p), 0, sizeof p);
    p.value = static_cast<typename P::value_type>(value);
    p.index = index;
    W w;
    std::memcpy(&w, &p, sizeof w);
    f(w);
  });
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

// The kernels of (type, op): the sum's are instantiated here, the other ops' in ring_allreduce_ops.cu.  The pair types
// have no sum: refused with the words of dispatch_op.
AllreduceKernels allreduce_kernels(ElemType type, ReduceOp op) {
  if (op != ReduceOp::kSum) return op_allreduce_kernels(type, op);
  HPCP_REQUIRE(reduce_op_takes(op, type), reduce_op_type_error(op, type));
  AllreduceKernels k{};
  dispatch_add_class(type, [&](auto tag) { k = allreduce_kernels_of<SumOp<decltype(tag)>, false, false>(); });
  return k;
}

// The fields RingDev and RingPullDev share.
template <class Dev>
Dev ring_dev(const RingArgs& args, size_t esz, size_t ce) {
  const size_t lanes = 16 / esz;
  Dev d{};
  d.va = static_cast<const uint4*>(args.va);
  d.vc = static_cast<uint4*>(args.vc);
  d.arrived_local = args.arrived_local;
  d.arrived_right = args.arrived_right;
  d.ack_local = args.ack_local;
  d.ack_left = args.ack_left;
  d.world = args.world;
  d.nvec = args.n / lanes;
  d.chunk_vec = ce / lanes;
  d.n_chunks = ring_num_chunks(args.n, ce, esz);
  d.epoch_base = args.epoch_base;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  return d;
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

void launch_accumulate(const void* va, void* vc, size_t n, ElemType type, cudaStream_t stream, ReduceOp op) {
  const size_t lanes = 16 / elem_size(type);
  const size_t nvec = n / lanes, tail = n % lanes;
  const int ctas = grid_for(std::max<size_t>(nvec, 1), 512, 132 * 4);
  // The sum keeps accumulate_kernel, whose scalar tail is typed: it is the timed step of ring-unfused, and running it
  // as combine_kernel<SumOp> would change that arm's instructions.
  if (op != ReduceOp::kSum) {
    const uint4* va_v = static_cast<const uint4*>(va);
    uint4* vc_v = static_cast<uint4*>(vc);
    const unsigned char* va_tail = static_cast<const unsigned char*>(va) + nvec * 16;
    unsigned char* vc_tail = static_cast<unsigned char*>(vc) + nvec * 16;
    launch_512(op_combine_kernel(type, op), ctas, stream, va_v, vc_v, nvec, va_tail, vc_tail, tail * elem_size(type));
    return;
  }
  HPCP_REQUIRE(reduce_op_takes(op, type), reduce_op_type_error(op, type));
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

void launch_init_pair(void* v, size_t n, double value, int index, ElemType type, cudaStream_t stream) {
  const int ctas = grid_for(n, 256, 132 * 8);
  with_pair_bits(type, value, index, [&](auto w) {
    using W = decltype(w);
    fill_pair_kernel<W><<<ctas, 256, 0, stream>>>(static_cast<W*>(v), n, w);
  });
  HPCP_CUDA(cudaGetLastError());
}

void launch_count_pair_mismatch(const void* v, size_t n, double value, int index, ElemType type,
                                unsigned long long* count, cudaStream_t stream) {
  const int ctas = grid_for(n, 256, 132 * 8);
  with_pair_bits(type, value, index, [&](auto w) {
    using W = decltype(w);
    count_pair_mismatch_kernel<W><<<ctas, 256, 0, stream>>>(static_cast<const W*>(v), n, w, count);
  });
  HPCP_CUDA(cudaGetLastError());
}

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
  const bool ack = args.n_slots == 2 && args.world > 3 && !args.pull;  // with P <= 3 no slot is ever written twice
  HPCP_REQUIRE(args.n_slots == 0 || args.n_slots == 2 || args.n_slots == args.world - 1,
               "ring: n_slots must be 0 (= world-1, no flow control) or 2 (double buffer + acks)");
  HPCP_REQUIRE(!ack || (args.ack_local != nullptr && args.ack_left != nullptr), "ring: n_slots=2 needs the ack words");
  HPCP_REQUIRE(!args.pull || args.world == 1 ||
                   (args.va_left != nullptr && (args.world == 2 || args.slots_left != nullptr)),
               "ring: the pull variant needs the left neighbour's VA and slots (peer-mapped)");
  HPCP_REQUIRE(!args.pull || args.n_slots != 2 || args.world <= 4 ||
                   (args.ack_local != nullptr && args.ack_left != nullptr),
               "ring: pull with n_slots=2 needs the ack words");
  const bool two_slots = args.n_slots == 2;  // slot index t % 2 even when no ack is ever needed (P <= 3)
  const void* kernel = allreduce_kernels(type, args.op).ring[args.pull][two_slots];
  if (args.pull) {
    RingPullDev d = ring_dev<RingPullDev>(args, esz, ce);
    d.va_left = static_cast<const uint4*>(args.va_left);
    d.slots_left = static_cast<const uint4*>(args.slots_left);
    d.slots_local = static_cast<uint4*>(args.slots_local);
    launch_512(kernel, ring_grid(kernel, d.n_chunks, ctas, device), stream, d);
  } else {
    RingDev d = ring_dev<RingDev>(args, esz, ce);
    d.slots_local = static_cast<const uint4*>(args.slots_local);
    d.slots_right = static_cast<uint4*>(args.slots_right);
    launch_512(kernel, ring_grid(kernel, d.n_chunks, ctas, device), stream, d);
  }
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
  // The all-gather phase only copies: every op shares the sum's kernel there, and a pair type (which has no sum) the one
  // of int: the body moves whole 16-byte vectors whatever the type.  The op is still checked against a pair type and
  // for maxloc / minloc, as in the other phases; the arithmetic types keep ignoring it there.
  const bool gather = args.phases == kRsAgAllGather;
  HPCP_REQUIRE(!gather || !(elem_type_is_pair(type) || reduce_op_on_pairs(args.op)) || reduce_op_takes(args.op, type),
               reduce_op_type_error(args.op, type));
  const ElemType ktype = gather && elem_type_is_pair(type) ? ElemType::kInt : type;
  const void* kernel = allreduce_kernels(ktype, gather ? ReduceOp::kSum : args.op).rsag;
  launch_512(kernel, ring_grid(kernel, d.n_chunks, ctas, device), stream, d);
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
  launch_512(allreduce_kernels(type, args.op).two_shot[two_shot_shape(args.world)], grid, stream, d);
  return grid;
}

int launch_reduce_scatter(const ReduceScatterArgs& args, ElemType type, int ctas, int device, cudaStream_t stream) {
  if (const char* why = reduce_scatter_refusal(args.world, args.n, type)) HPCP_FAIL(why);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "reduce-scatter: rank out of range");
  const void* kernel = allreduce_kernels(type, args.op).reduce_scatter[two_shot_shape(args.world)];  // op refusals
  const size_t seg_bytes = args.n * elem_size(type);
  HPCP_REQUIRE(!byte_ranges_overlap(args.send[args.rank], seg_bytes * static_cast<size_t>(args.world), args.recv,
                                    seg_bytes),
               kReduceScatterOverlapError);
  TwoShotDev d{};  // two-shot's block: va = the send buffers, vc[rank] = my receive buffer (two_shot_body's kScatter)
  for (int p = 0; p < args.world; ++p) {
    d.va[p] = static_cast<const uint4*>(args.send[p]);
    d.pads[p] = args.pads[p];
  }
  d.vc[args.rank] = static_cast<uint4*>(args.recv);
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.slice_vec = seg_bytes / 16;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  const int sms = device_sm_count(device);
  const int grid = grid_for(d.slice_vec, 512, ctas > 0 ? ctas : sms * 2);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
  launch_512(kernel, grid, stream, d);
  return grid;
}

int launch_allreduce_nvls(const NvlsArgs& args, ElemType type, int ctas, int device,
                          cudaStream_t stream) {
  HPCP_REQUIRE(args.world >= 1 && args.world <= kApiMaxRanks, "nvls: world out of range");
  HPCP_REQUIRE(args.op == ReduceOp::kSum,
               "nvls: only op=sum is supported (multimem.ld_reduce min/max is not wired); use two-shot for prod/min/max");
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
  const int sms = device_sm_count(device);
  // Default grid: 32 CTAs.  The in-switch reduction saturates at modest request parallelism and more requesters only
  // queue in the switch.  HPCP_NVLS_CTAS_PER_SM / --ctas override.
  const int grid = grid_for(std::max<size_t>(d.slice_vec, 1), 512, ctas > 0 ? ctas : per_sm > 0 ? sms * per_sm : 32);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
  const bool f32 = type == ElemType::kFloat;
  const void* kernel =
      unroll == 8 ? (f32 ? kernel_ptr(nvls_kernel<float, 8, 512>) : kernel_ptr(nvls_kernel<int, 8, 512>))
                  : (f32 ? kernel_ptr(nvls_kernel<float, 4, 512>) : kernel_ptr(nvls_kernel<int, 4, 512>));
  launch_512(kernel, grid, stream, d);
  return grid;
}

}  // namespace hpcp
