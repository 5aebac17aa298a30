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

template <bool kPull>
__global__ void __launch_bounds__(512) all_to_all_kernel(const __grid_constant__ AllToAllDev a) {
  constexpr int U = kA2aVectors;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t bv = a.block_vec;
  size_t off = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;  // offset in the current block
  for (int j = 0; j < a.world; ++j) {
    const int p = (a.rank + 1 + j) % a.world;
    const uint4* src = kPull ? a.send[p] + a.rank * bv : a.send[a.rank] + p * bv;
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

}  // namespace hpcp
