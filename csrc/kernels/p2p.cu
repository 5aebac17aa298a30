// K-p2p: GPU<->GPU data movement over NVLink peer mappings, from inside a kernel.
//
// Replaces the transports of the reference's p2p benchmark:
//   MPI_Isend/Irecv/Waitall  p2p/peer2pear.cpp:32-44  -> rendezvous: wait "ready" word, move, publish "done"
//   MPI_Put + MPI_Win_fence  p2p/peer2pear.cpp:76-81  -> move, publish "done"
//   (MPI_Get, absent upstream, requested by BASELINE.json) -> peer loads
// plus the payload fill (peer2pear.cpp:8-17) and receiver check (:55-63), both
// moved onto the device and made exact.
//
// Two engines:
//   LdSt : every thread keeps UNROLL independent 128-bit loads in flight, then
//          stores them (coalesced 512 B per warp per access).
//   Tma  : ONE elected thread per CTA streams tiles global->smem->global with
//          cp.async.bulk (SASS: UBLKCP) through a ring of mbarrier-tracked smem
//          stages.  It needs no registers/LSU of the other warps, which is what
//          lets the fused bench kernels run math next to the copy.
#include "api.h"

#include <algorithm>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "payload.h"

namespace hpcp {

namespace {

// Prologue shared by the data movers: one thread waits for the epoch, the CTA
// learns the outcome through smem.
__device__ __forceinline__ bool prologue_wait(const SyncOps& sync) {
  if (sync.wait_flag == nullptr) return true;
  __shared__ int ok_s;
  if (threadIdx.x == 0)
    ok_s = wait_epoch(sync.wait_flag, sync.wait_epoch, sync.timeout_ns, sync.status) ? 1 : 0;
  __syncthreads();
  return ok_s != 0;
}

__device__ __forceinline__ void epilogue_signal(const SyncOps& sync) {
  if (sync.ticket == nullptr) return;
  last_cta_publish(sync.ticket, sync.ticket_base + gridDim.x, sync.signal_flag,
                   sync.signal_epoch);
}

// ------------------------------------------------------------ LdSt engine ----
// V = uint4 (LDG/STG.128) or ptx::U32x8 (two LDG/STG.128 per thread).
template <typename V, bool kPeerSrc>
__device__ __forceinline__ V ld_vec(const V* p);
template <>
__device__ __forceinline__ uint4 ld_vec<uint4, false>(const uint4* p) { return ptx::ld_stream_v4(p); }
template <>
__device__ __forceinline__ uint4 ld_vec<uint4, true>(const uint4* p) { return ptx::ld_peer_v4(p); }
template <>
__device__ __forceinline__ ptx::U32x8 ld_vec<ptx::U32x8, false>(const ptx::U32x8* p) { return ptx::ld_stream_v8(p); }
template <>
__device__ __forceinline__ ptx::U32x8 ld_vec<ptx::U32x8, true>(const ptx::U32x8* p) { return ptx::ld_weak_v8(p); }
__device__ __forceinline__ void st_vec(uint4* p, const uint4& v) { ptx::st_stream_v4(p, v); }
__device__ __forceinline__ void st_vec(ptx::U32x8* p, const ptx::U32x8& v) { ptx::st_stream_v8(p, v); }

template <typename V, int U, bool kPeerSrc>
__global__ void __launch_bounds__(1024)
    copy_ldst_kernel(V* __restrict__ dst, const V* __restrict__ src, size_t nvec, size_t tail_bytes,
                     int blocked, SyncOps sync) {
  if (!prologue_wait(sync)) return;

  // interleaved: vector i of batch k is handled by thread (i mod stride); blocked: every CTA
  // owns one contiguous range (sequential NVLink / HBM pages per CTA).
  size_t begin, end, stride;
  if (blocked) {
    const size_t per = (nvec + gridDim.x - 1) / gridDim.x;
    begin = static_cast<size_t>(blockIdx.x) * per;
    end = begin + per < nvec ? begin + per : nvec;
    stride = blockDim.x;
    begin += threadIdx.x;
  } else {
    stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    begin = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    end = nvec;
  }
  size_t i = begin;
  for (; i + (U - 1) * stride < end; i += U * stride) {
    V v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) v[k] = ld_vec<V, kPeerSrc>(src + i + k * stride);
#pragma unroll
    for (int k = 0; k < U; ++k) st_vec(dst + i + k * stride, v[k]);
  }
  for (; i < end; i += stride) st_vec(dst + i, ld_vec<V, kPeerSrc>(src + i));
  if (tail_bytes != 0 && blockIdx.x == 0 && threadIdx.x < tail_bytes) {
    const unsigned char* s = reinterpret_cast<const unsigned char*>(src + nvec);
    unsigned char* d = reinterpret_cast<unsigned char*>(dst + nvec);
    d[threadIdx.x] = s[threadIdx.x];
  }
  epilogue_signal(sync);
}

// ------------------------------------------------------------- TMA engine ----
// Dynamic smem: [stages][stage_bytes] data | [stages] mbarriers.
__global__ void __launch_bounds__(32)
    copy_tma_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src,
                    size_t bytes16 /*multiple of 16*/, size_t tail_bytes, uint32_t stage_bytes,
                    int stages, SyncOps sync) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(stages) * stage_bytes);

  if (!prologue_wait(sync)) return;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) ptx::mbar_init(&full[s], 1);
    ptx::fence_mbar_init();

    const size_t n_tiles_total = (bytes16 + stage_bytes - 1) / stage_bytes;
    // Tiles owned by this CTA: blockIdx.x, +gridDim.x, ...
    const size_t n = n_tiles_total > blockIdx.x
                         ? (n_tiles_total - blockIdx.x + gridDim.x - 1) / gridDim.x
                         : 0;
    auto tile_off = [&](size_t j) {
      return (static_cast<size_t>(blockIdx.x) + j * gridDim.x) * stage_bytes;
    };
    auto tile_len = [&](size_t j) {
      const size_t off = tile_off(j);
      return static_cast<uint32_t>(bytes16 - off < stage_bytes ? bytes16 - off : stage_bytes);
    };
    auto issue_load = [&](size_t j) {
      const int st = static_cast<int>(j % stages);
      const uint32_t len = tile_len(j);
      ptx::mbar_arrive_expect_tx(&full[st], len);
      ptx::bulk_g2s(smem + static_cast<size_t>(st) * stage_bytes, src + tile_off(j), len, &full[st]);
    };

    const size_t lookahead = static_cast<size_t>(stages - 1);
    for (size_t j = 0; j < lookahead && j < n; ++j) issue_load(j);
    for (size_t j = 0; j < n; ++j) {
      const int st = static_cast<int>(j % stages);
      ptx::mbar_wait(&full[st], static_cast<uint32_t>((j / stages) & 1));
      ptx::bulk_s2g(dst + tile_off(j), smem + static_cast<size_t>(st) * stage_bytes, tile_len(j));
      ptx::bulk_commit();
      const size_t nxt = j + lookahead;
      if (nxt < n) {
        // Stage of tile `nxt` was last read by store group j-1: allow only the
        // newest group (j) to still be reading its smem source.
        ptx::bulk_wait_read<1>();
        issue_load(nxt);
      }
    }
    ptx::bulk_wait<0>();  // all bulk stores performed
    asm volatile("fence.proxy.async;" ::: "memory");
    if (tail_bytes != 0 && blockIdx.x == 0)
      for (size_t t = 0; t < tail_bytes; ++t) dst[bytes16 + t] = src[bytes16 + t];
  }
  epilogue_signal(sync);
}

// ------------------------------------------------------- fill and verify ----
__global__ void fill_pattern_kernel(uint32_t* __restrict__ dst, size_t n, uint32_t seed) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = pattern_word(i, seed);
}

__global__ void verify_pattern_kernel(const uint32_t* __restrict__ data, size_t n, uint32_t seed,
                                      unsigned long long* mismatch_count,
                                      unsigned long long* word_sum, SyncOps sync) {
  if (!prologue_wait(sync)) return;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0, sum = 0;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    // Volatile-free but fresh: the buffer was written by a peer; kernel-boundary or
    // the acquire in prologue_wait ordered those writes before these loads.
    const uint32_t got = __ldcg(data + i);
    bad += (got != pattern_word(i, seed));
    sum += got;
  }
  for (int off = 16; off > 0; off >>= 1) {
    bad += __shfl_xor_sync(0xffffffffu, bad, off);
    sum += __shfl_xor_sync(0xffffffffu, sum, off);
  }
  if ((threadIdx.x & 31) == 0) {
    if (bad) atomicAdd(mismatch_count, bad);
    if (word_sum != nullptr) atomicAdd(word_sum, sum);
  }
  if (bad && sync.status != nullptr && (threadIdx.x & 31) == 0)
    ptx::st_relaxed_sys(sync.status, kStatusMismatch);
}

// ---------------------------------------------------------------- signals ----
__global__ void signal_kernel(uint32_t* flag, uint32_t epoch) { publish_epoch(flag, epoch); }

__global__ void wait_kernel(const uint32_t* flag, uint32_t epoch, uint64_t timeout_ns,
                            uint32_t* status) {
  wait_epoch(flag, epoch, timeout_ns, status);
}

struct PadList {
  uint32_t* pad[kApiMaxRanks];
};

__global__ void barrier_all_kernel(PadList pads, int rank, int world, uint32_t epoch,
                                   uint64_t timeout_ns, uint32_t* status) {
  const int t = threadIdx.x;
  if (t < world) {
    // Everything this stream did before the barrier is ordered by the kernel
    // boundary; the fence makes it visible system-wide before the arrival word.
    publish_epoch(pads.pad[t] + kPadBarrier + rank, epoch);
    wait_epoch(pads.pad[rank] + kPadBarrier + t, epoch, timeout_ns, status);
  }
}

}  // namespace

int device_sm_count(int device) {
  static int cache[64] = {0};
  if (device >= 0 && device < 64 && cache[device] > 0) return cache[device];
  int n = 0;
  HPCP_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device));
  if (device >= 0 && device < 64) cache[device] = n;
  return n;
}

void launch_signal(uint32_t* flag, uint32_t epoch, cudaStream_t stream) {
  signal_kernel<<<1, 1, 0, stream>>>(flag, epoch);
  HPCP_CUDA(cudaGetLastError());
}

void launch_wait(const uint32_t* flag, uint32_t epoch, uint64_t timeout_ns, uint32_t* status,
                 cudaStream_t stream) {
  wait_kernel<<<1, 1, 0, stream>>>(flag, epoch, timeout_ns, status);
  HPCP_CUDA(cudaGetLastError());
}

void launch_barrier_all(uint32_t* const* pads, int rank, int world, uint32_t epoch,
                        uint64_t timeout_ns, uint32_t* status, cudaStream_t stream) {
  HPCP_REQUIRE(world >= 1 && world <= kApiMaxRanks, "barrier_all: world out of range");
  PadList pl{};
  for (int r = 0; r < world; ++r) pl.pad[r] = pads[r];
  barrier_all_kernel<<<1, 32, 0, stream>>>(pl, rank, world, epoch, timeout_ns, status);
  HPCP_CUDA(cudaGetLastError());
}

namespace {

template <typename V, bool kPeerSrc>
void launch_ldst(void* dst, const void* src, size_t nvec, size_t tail, int unroll, int ctas,
                 int threads, int blocked, const SyncOps& sync, cudaStream_t stream) {
  V* d = static_cast<V*>(dst);
  const V* s = static_cast<const V*>(src);
  switch (unroll) {
    case 1: copy_ldst_kernel<V, 1, kPeerSrc><<<ctas, threads, 0, stream>>>(d, s, nvec, tail, blocked, sync); break;
    case 2: copy_ldst_kernel<V, 2, kPeerSrc><<<ctas, threads, 0, stream>>>(d, s, nvec, tail, blocked, sync); break;
    case 8:
      if constexpr (sizeof(V) == 16) {  // 8 x 256-bit would not fit 64 registers/thread
        copy_ldst_kernel<V, 8, kPeerSrc><<<ctas, threads, 0, stream>>>(d, s, nvec, tail, blocked, sync);
        break;
      }
      [[fallthrough]];
    default: copy_ldst_kernel<V, 4, kPeerSrc><<<ctas, threads, 0, stream>>>(d, s, nvec, tail, blocked, sync); break;
  }
}

}  // namespace

int launch_copy(void* dst, const void* src, size_t bytes, bool src_is_peer, CopyEngine engine,
                const CopyTuning& tune, const SyncOps& sync, int device, cudaStream_t stream) {
  HPCP_REQUIRE((reinterpret_cast<uintptr_t>(dst) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(src) & 15) == 0,
               "launch_copy: pointers must be 16-byte aligned");
  HPCP_REQUIRE(sync.signal_flag == nullptr || sync.ticket != nullptr,
               "launch_copy: a signal needs a ticket counter");
  const int sms = device_sm_count(device);
  const size_t nvec = bytes / 16;
  const size_t tail = bytes % 16;
  int ctas = 0;

  if (engine == CopyEngine::kLdSt) {
    const int threads = tune.threads > 0 ? std::min(tune.threads, 1024) : 512;
    const int unroll = tune.unroll > 0 ? tune.unroll : 4;
    const bool wide = tune.vec_bytes == 32 &&
                      (reinterpret_cast<uintptr_t>(dst) & 31) == 0 &&
                      (reinterpret_cast<uintptr_t>(src) & 31) == 0;
    const size_t vb = wide ? 32 : 16;
    const size_t nv = bytes / vb;
    const size_t tl = bytes % vb;
    const size_t per_cta = static_cast<size_t>(threads) * unroll;
    const size_t want = std::max<size_t>(1, (nv + per_cta - 1) / per_cta);
    const int cap = tune.ctas > 0 ? tune.ctas : sms * 2;
    ctas = static_cast<int>(std::min<size_t>(want, static_cast<size_t>(cap)));
    HPCP_REQUIRE(tl < static_cast<size_t>(threads), "launch_copy: tail larger than the CTA");
    if (wide) {
      if (src_is_peer)
        launch_ldst<ptx::U32x8, true>(dst, src, nv, tl, unroll, ctas, threads, tune.blocked, sync, stream);
      else
        launch_ldst<ptx::U32x8, false>(dst, src, nv, tl, unroll, ctas, threads, tune.blocked, sync, stream);
    } else {
      if (src_is_peer)
        launch_ldst<uint4, true>(dst, src, nv, tl, unroll, ctas, threads, tune.blocked, sync, stream);
      else
        launch_ldst<uint4, false>(dst, src, nv, tl, unroll, ctas, threads, tune.blocked, sync, stream);
    }
  } else {
    const uint32_t stage_bytes = static_cast<uint32_t>((tune.stage_kb > 0 ? tune.stage_kb : 16) * 1024);
    const int stages = tune.stages > 0 ? tune.stages : 8;
    HPCP_REQUIRE(stages >= 2, "launch_copy: TMA engine needs >= 2 stages");
    const size_t smem = static_cast<size_t>(stages) * stage_bytes + static_cast<size_t>(stages) * 8;
    HPCP_REQUIRE(smem <= 227 * 1024, "launch_copy: TMA stages exceed 227 KiB of shared memory");
    const size_t bytes16 = nvec * 16;
    const size_t tiles = std::max<size_t>(1, (bytes16 + stage_bytes - 1) / stage_bytes);
    // CTAs per SM limited by smem; default one resident wave.
    const int per_sm = std::max(1, static_cast<int>((227 * 1024) / smem));
    const int cap = tune.ctas > 0 ? tune.ctas : sms * std::min(per_sm, 2);
    ctas = static_cast<int>(std::min<size_t>(tiles, static_cast<size_t>(cap)));
    HPCP_ENABLE_SMEM(copy_tma_kernel, smem);
    copy_tma_kernel<<<ctas, 32, smem, stream>>>(static_cast<unsigned char*>(dst),
                                                static_cast<const unsigned char*>(src), bytes16,
                                                tail, stage_bytes, stages, sync);
  }
  HPCP_CUDA(cudaGetLastError());
  return ctas;
}

void launch_fill_pattern(uint32_t* dst, size_t n_words, uint32_t seed, cudaStream_t stream) {
  const int threads = 256;
  const int ctas = static_cast<int>(std::min<size_t>((n_words + threads - 1) / threads, 132 * 8));
  fill_pattern_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(dst, n_words, seed);
  HPCP_CUDA(cudaGetLastError());
}

void launch_verify_pattern(const uint32_t* data, size_t n_words, uint32_t seed,
                           unsigned long long* mismatch_count, unsigned long long* word_sum,
                           const uint32_t* wait_flag, uint32_t wait_epoch, uint64_t timeout_ns,
                           uint32_t* status, cudaStream_t stream) {
  SyncOps sync;
  sync.wait_flag = wait_flag;
  sync.wait_epoch = wait_epoch;
  sync.timeout_ns = timeout_ns;
  sync.status = status;
  const int threads = 256;
  // All CTAs may spin in the prologue, so keep the grid within one resident wave.
  const int ctas = static_cast<int>(std::min<size_t>((n_words + threads - 1) / threads, 132 * 4));
  verify_pattern_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(data, n_words, seed,
                                                                  mismatch_count, word_sum, sync);
  HPCP_CUDA(cudaGetLastError());
}

}  // namespace hpcp
