// All-to-all (↔ MPI_Alltoall with equal blocks, ncclAllToAll, torch.distributed.all_to_all_single) in ONE launch per
// rank over peer mappings.  Every rank holds a send and a receive buffer of P blocks of B bytes; afterwards block p of
// rank r's receive buffer is a byte copy of block r of rank p's send buffer.
//
//   push (kPull = false): rank r loads its own send block q and stores it into slot r of rank q's receive buffer;
//   pull (kPull = true):  rank r loads slot r of rank p's send buffer and stores it into its own receive block p.
//
// The walk is staggered: block j of the walk is peer (rank + 1 + j) % P (the rule of tile_order.h), so at any moment
// the P ranks address P different peers, and the local block comes last.  The P blocks are walked as ONE grid-stride
// loop over their concatenation: a thread's offset carries over from one block into the next, so small blocks keep
// every CTA busy and no index is divided.  Inside a block each thread keeps kA2aVectors independent 128-bit loads in
// flight; a tail loop takes what is left of a block.  The launch ends with two-shot's grid_then_node_barrier: when the
// kernel completes, every peer's bytes have landed in my receive buffer and every peer has finished reading my send
// buffer.
#include "alltoallv_plan.h"
#include "ring_allreduce.cuh"

namespace hpcp {

namespace {

// Independent 16-byte vectors in flight per thread and trip: two-shot's U at up to 4 ranks.
constexpr int kA2aVectors = 4;

struct AllToAllDev {
  const uint4* send[kApiMaxRanks];
  uint4* recv[kApiMaxRanks];
  uint32_t* pads[kApiMaxRanks];
  uint32_t* ticket;
  uint32_t ticket_target;
  int rank;
  int world;
  size_t block_vec;  // 16-byte vectors per block
  uint32_t barrier_epoch;
  uint64_t timeout_ns;
  uint32_t* status;
};

// kGather: the all-gather, the same walk with a source stride of 0.  Every rank's send buffer is ONE block, and block p
// of every receive buffer is rank p's: push stores my block into slot `rank` of every rank's receive buffer, pull loads
// rank p's block into my slot p.
template <bool kPull, bool kGather>
__device__ __forceinline__ void a2a_walk(const AllToAllDev& a) {
  constexpr int U = kA2aVectors;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t bv = a.block_vec;
  size_t off = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // offset in the current block
  for (int j = 0; j < a.world; ++j) {
    const int p = (a.rank + 1 + j) % a.world;
    const uint4* src;
    if constexpr (kGather)
      src = kPull ? a.send[p] : a.send[a.rank];
    else
      src = kPull ? a.send[p] + a.rank * bv : a.send[a.rank] + p * bv;
    uint4* dst = kPull ? a.recv[a.rank] + p * bv : a.recv[p] + a.rank * bv;
    for (; off + (U - 1) * stride < bv; off += U * stride) {
      uint4 x[U];
#pragma unroll
      for (int u = 0; u < U; ++u) x[u] = kPull ? ptx::ld_peer_v4(src + off + u * stride) : ptx::ld_stream_v4(src + off + u * stride);
#pragma unroll
      for (int u = 0; u < U; ++u) ptx::st_stream_v4(dst + off + u * stride, x[u]);
    }
    for (; off < bv; off += stride)
      ptx::st_stream_v4(dst + off, kPull ? ptx::ld_peer_v4(src + off) : ptx::ld_stream_v4(src + off));
    off -= bv;  // the same thread goes on in the next block of the walk
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch, a.timeout_ns, a.status);
}

template <bool kPull>
__global__ void __launch_bounds__(512) all_to_all_kernel(const __grid_constant__ AllToAllDev a) {
  a2a_walk<kPull, false>(a);
}

template <bool kPull>
__global__ void __launch_bounds__(512) all_gather_kernel(const __grid_constant__ AllToAllDev a) {
  a2a_walk<kPull, true>(a);
}

// ---------------------------------------------------------------------------------------------- all-to-all-v ----
// Every CTA loads the world x world count matrix over peer memory into shared memory (one count per thread), judges
// it with the rules of alltoallv_plan.h (thread p takes row p, thread world+q column q) and, if it is accepted, walks
// the world segments of its rank in the staggered order above: push stores my segment for p at its packed row in p's
// receive buffer, pull loads p's segment for me into my receive buffer.  The walk is the equal-block kernel's
// grid-stride loop over the concatenation of the segments; `off -= seg` carries a thread's offset into the next
// segment whatever the segments' sizes, and an empty segment costs one comparison.  Every CTA reaches the same verdict
// from the same matrix, so a refused launch moves nothing anywhere, and the node barrier ends every launch.
struct AllToAllVDev {
  const uint4* send[kApiMaxRanks];
  uint4* recv[kApiMaxRanks];
  const int64_t* counts[kApiMaxRanks];
  uint32_t* pads[kApiMaxRanks];
  int64_t* recv_counts;
  uint32_t* verdict;
  uint32_t* ticket;
  uint32_t ticket_target;
  int rank;
  int world;
  size_t row_vec;  // 16-byte vectors per row
  int64_t send_capacity_rows;
  int64_t recv_capacity_rows;
  uint32_t barrier_epoch;
  uint64_t timeout_ns;
  uint32_t* status;
};

// The peer's counts may have been written by a kernel of the previous step: coherent with the remote writer, no .nc.
__device__ __forceinline__ int64_t ld_count(const int64_t* p) {
  int64_t v;
  asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

template <bool kPull>
__global__ void __launch_bounds__(512) all_to_all_v_kernel(const __grid_constant__ AllToAllVDev a) {
  constexpr int U = kA2aVectors;
  __shared__ int64_t m[kApiMaxRanks * kApiMaxRanks];
  __shared__ size_t seg_vec[kApiMaxRanks], src_vec[kApiMaxRanks], dst_vec[kApiMaxRanks];
  __shared__ uint32_t broken;  // bit k: rule k is broken in some row or column
  const int P = a.world, t = threadIdx.x;
  if (t == 0) broken = 0;
  if (t < P * P) m[t] = ld_count(a.counts[t / P] + t % P);
  __syncthreads();
  if (t < P)
    atomicOr(&broken, 1u << a2av_row_rule(m, P, t, a.send_capacity_rows));
  else if (t < 2 * P)
    atomicOr(&broken, 1u << a2av_col_rule(m, P, t - P, a.recv_capacity_rows));
  __syncthreads();
  const uint32_t verdict = a2av_first_rule(broken);
  if (blockIdx.x == 0) {
    if (t < P) a.recv_counts[t] = m[t * P + a.rank];
    if (t == 0) *a.verdict = verdict;
  }
  if (verdict == kA2avAccepted) {  // the same in every thread of the grid
    if (t < P) {                   // segment j of the walk: sender s -> receiver r
      const int p = (a.rank + 1 + t) % P, s = kPull ? p : a.rank, r = kPull ? a.rank : p;
      seg_vec[t] = static_cast<size_t>(m[s * P + r]) * a.row_vec;
      src_vec[t] = static_cast<size_t>(a2av_send_offset(m, P, s, r)) * a.row_vec;
      dst_vec[t] = static_cast<size_t>(a2av_recv_offset(m, P, s, r)) * a.row_vec;
    }
    __syncthreads();
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    size_t off = static_cast<size_t>(blockIdx.x) * blockDim.x + t;  // offset in the current segment
    for (int j = 0; j < P; ++j) {
      const int p = (a.rank + 1 + j) % P;
      const size_t sv = seg_vec[j];
      const uint4* src = (kPull ? a.send[p] : a.send[a.rank]) + src_vec[j];
      uint4* dst = (kPull ? a.recv[a.rank] : a.recv[p]) + dst_vec[j];
      for (; off + (U - 1) * stride < sv; off += U * stride) {
        uint4 x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) x[u] = kPull ? ptx::ld_peer_v4(src + off + u * stride) : ptx::ld_stream_v4(src + off + u * stride);
#pragma unroll
        for (int u = 0; u < U; ++u) ptx::st_stream_v4(dst + off + u * stride, x[u]);
      }
      for (; off < sv; off += stride)
        ptx::st_stream_v4(dst + off, kPull ? ptx::ld_peer_v4(src + off) : ptx::ld_stream_v4(src + off));
      off -= sv;  // the same thread goes on in the next segment of the walk
    }
  }
  grid_then_node_barrier(a.ticket, a.ticket_target, a.pads, a.rank, a.world, a.barrier_epoch, a.timeout_ns, a.status);
}

}  // namespace

const char* all_to_all_refusal(int world, size_t block_bytes) {
  if (block_bytes == 0 || block_bytes % 16 != 0) return kAllToAllBlockError;
  if (world < 1 || world > kApiMaxRanks) return kAllToAllWorldError;
  return nullptr;
}

int launch_all_to_all(const AllToAllArgs& args, int ctas, int device, cudaStream_t stream) {
  if (const char* why = all_to_all_refusal(args.world, args.block_bytes)) HPCP_FAIL(why);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "all-to-all: rank out of range");
  const size_t bytes = args.block_bytes * static_cast<size_t>(args.world);
  const auto s = reinterpret_cast<uintptr_t>(args.send[args.rank]), r = reinterpret_cast<uintptr_t>(args.recv[args.rank]);
  HPCP_REQUIRE(s + bytes <= r || r + bytes <= s, kAllToAllOverlapError);
  AllToAllDev d{};
  for (int p = 0; p < args.world; ++p) {
    d.send[p] = static_cast<const uint4*>(args.send[p]);
    d.recv[p] = static_cast<uint4*>(args.recv[p]);
    d.pads[p] = args.pads[p];
  }
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.block_vec = args.block_bytes / 16;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  const int sms = device_sm_count(device);
  const int grid = grid_for(d.block_vec * args.world, 512, ctas > 0 ? ctas : sms * 2);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
  const void* kernel = args.pull ? kernel_ptr(all_to_all_kernel<true>) : kernel_ptr(all_to_all_kernel<false>);
  launch_512(kernel, grid, stream, d);
  return grid;
}

int launch_all_gather(const AllGatherArgs& args, int ctas, int device, cudaStream_t stream) {
  if (const char* why = all_gather_refusal(args.world, args.block_bytes)) HPCP_FAIL(why);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "all-gather: rank out of range");
  HPCP_REQUIRE(!byte_ranges_overlap(args.send[args.rank], args.block_bytes, args.recv[args.rank],
                                    args.block_bytes * static_cast<size_t>(args.world)),
               kAllGatherOverlapError);
  AllToAllDev d{};
  for (int p = 0; p < args.world; ++p) {
    d.send[p] = static_cast<const uint4*>(args.send[p]);
    d.recv[p] = static_cast<uint4*>(args.recv[p]);
    d.pads[p] = args.pads[p];
  }
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.block_vec = args.block_bytes / 16;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  const int sms = device_sm_count(device);
  const int grid = grid_for(d.block_vec * args.world, 512, ctas > 0 ? ctas : sms * 2);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
  const void* kernel = args.pull ? kernel_ptr(all_gather_kernel<true>) : kernel_ptr(all_gather_kernel<false>);
  launch_512(kernel, grid, stream, d);
  return grid;
}

const char* all_to_all_v_refusal(int world, size_t row_bytes, int64_t send_capacity_rows, int64_t recv_capacity_rows) {
  if (row_bytes == 0 || row_bytes % 16 != 0) return kAllToAllVRowError;
  if (world < 1 || world > kApiMaxRanks) return kAllToAllWorldError;
  if (send_capacity_rows <= 0 || recv_capacity_rows <= 0) return kAllToAllVCapacityError;
  return nullptr;
}

const char* all_to_all_v_verdict_words(uint32_t verdict) {
  switch (verdict) {
    case kA2avAccepted: return "";
    case kA2avNegative: return "all-to-all-v: a count is negative";
    case kA2avSendCapacity: return "all-to-all-v: a rank's counts exceed the send capacity";
    case kA2avRecvCapacity: return "all-to-all-v: the counts into a rank exceed the receive capacity";
    default: return "all-to-all-v: unknown verdict";
  }
}

int launch_all_to_all_v(const AllToAllVArgs& args, int ctas, int device, cudaStream_t stream) {
  if (const char* why = all_to_all_v_refusal(args.world, args.row_bytes, args.send_capacity_rows,
                                             args.recv_capacity_rows))
    HPCP_FAIL(why);
  HPCP_REQUIRE(args.rank >= 0 && args.rank < args.world, "all-to-all-v: rank out of range");
  const auto disjoint = [](const void* x, size_t nx, const void* y, size_t ny) {
    const auto a = reinterpret_cast<uintptr_t>(x), b = reinterpret_cast<uintptr_t>(y);
    return a + nx <= b || b + ny <= a;
  };
  HPCP_REQUIRE(disjoint(args.send[args.rank], static_cast<size_t>(args.send_capacity_rows) * args.row_bytes,
                        args.recv[args.rank], static_cast<size_t>(args.recv_capacity_rows) * args.row_bytes),
               kAllToAllOverlapError);
  const size_t counts_bytes = sizeof(int64_t) * static_cast<size_t>(args.world);
  HPCP_REQUIRE(disjoint(args.counts[args.rank], counts_bytes, args.recv_counts, counts_bytes),
               kAllToAllVCountsOverlapError);
  AllToAllVDev d{};
  for (int p = 0; p < args.world; ++p) {
    d.send[p] = static_cast<const uint4*>(args.send[p]);
    d.recv[p] = static_cast<uint4*>(args.recv[p]);
    d.counts[p] = args.counts[p];
    d.pads[p] = args.pads[p];
  }
  d.recv_counts = args.recv_counts;
  d.verdict = args.verdict;
  d.ticket = args.ticket;
  d.rank = args.rank;
  d.world = args.world;
  d.row_vec = args.row_bytes / 16;
  d.send_capacity_rows = args.send_capacity_rows;
  d.recv_capacity_rows = args.recv_capacity_rows;
  d.barrier_epoch = args.barrier_epoch;
  d.timeout_ns = args.timeout_ns;
  d.status = args.status;
  // The host does not know how many rows move: size the grid for the most this rank can move (its send capacity
  // when it pushes, its receive capacity when it pulls).
  const int sms = device_sm_count(device);
  const int64_t cap_rows = args.pull ? args.recv_capacity_rows : args.send_capacity_rows;
  const int grid = grid_for(static_cast<size_t>(cap_rows) * d.row_vec, 512, ctas > 0 ? ctas : sms * 2);
  d.ticket_target = args.ticket_base + static_cast<uint32_t>(grid);
  const void* kernel = args.pull ? kernel_ptr(all_to_all_v_kernel<true>) : kernel_ptr(all_to_all_v_kernel<false>);
  launch_512(kernel, grid, stream, d);
  return grid;
}

}  // namespace hpcp
