// K-fused-triad-put: fused compute + one-directional ring put (round 1's flagship; K-halo in halo_stencil.cu, where
// every step consumes what the neighbours produced, is the flagship since round 2).
//
// The reference never overlaps compute with communication: its miniapp runs
// "kernel; wait; MPI_Send/Recv; wait" (allreduce-mpi-sycl.cpp:176-181, whose
// header calls the kernel "triad + send/recv", :1-4) and its concurrency bench
// only asks the runtime to overlap separately submitted commands
// (concurency/bench_sycl.cpp:84-121).  Here the stream triad
//        a[i] = b[i] + s * c[i]
// and the P2P put of `a` to a neighbour GPU are ONE kernel: each result vector
// is produced once in registers (LdSt engine) or once in shared memory (TMA
// engine) and written to BOTH the local array and the peer's receive buffer
// over NVLink.  The put costs no extra HBM read, there is no second launch, no
// MPI/NCCL/cudaMemcpy, and arrival is published to the peer with a
// release-scoped epoch word in the same launch.
//
// TMA engine layout (warp specialised, one CTA per SM):
//   warp 0 / lane 0 : DMA thread — cp.async.bulk b,c tiles -> smem stage
//                     (mbarrier complete_tx), later cp.async.bulk smem -> a_local
//                     and smem -> a_peer for the computed tile.
//   warps 1..4      : math — wait full[stage], a = b + s*c in place in smem,
//                     fence.proxy.async, arrive on computed[stage].
#include "api.h"

#include <algorithm>

#include "../common/cuda_check.h"
#include "../common/signal.cuh"
#include "payload.h"

namespace hpcp {

namespace {

__device__ __forceinline__ float4 triad4(const float4& b, const float4& c, float s) {
  return make_float4(fmaf(s, c.x, b.x), fmaf(s, c.y, b.y), fmaf(s, c.z, b.z), fmaf(s, c.w, b.w));
}

__device__ __forceinline__ bool cta_prologue_wait(const SyncOps& sync) {
  if (sync.wait_flag == nullptr) return true;
  __shared__ int ok_s;
  if (threadIdx.x == 0)
    ok_s = wait_epoch(sync.wait_flag, sync.wait_epoch, sync.timeout_ns, sync.status) ? 1 : 0;
  __syncthreads();
  return ok_s != 0;
}

// Publish "my put landed" on the peer (last CTA) and, on CTA 0, wait for the
// neighbour's put into *my* buffer, so kernel completion == exchange complete.
__device__ __forceinline__ void cta_epilogue(const SyncOps& sync, const uint32_t* arrive_flag,
                                             uint32_t arrive_epoch) {
  if (sync.ticket != nullptr)
    last_cta_publish(sync.ticket, sync.ticket_base + gridDim.x, sync.signal_flag,
                     sync.signal_epoch);
  if (arrive_flag != nullptr && blockIdx.x == 0 && threadIdx.x == 0)
    wait_epoch(arrive_flag, arrive_epoch, sync.timeout_ns, sync.status);
}

// ------------------------------------------------------------ LdSt engine ----
// V = uint4 (4 floats, LDG/STG.128) or ptx::U32x8 (8 floats, two LDG/STG.128).
__device__ __forceinline__ uint4 ld_in(const uint4* p) { return ptx::ld_stream_v4(p); }
__device__ __forceinline__ ptx::U32x8 ld_in(const ptx::U32x8* p) { return ptx::ld_stream_v8(p); }
__device__ __forceinline__ void st_out(uint4* p, const uint4& v) { ptx::st_stream_v4(p, v); }
__device__ __forceinline__ void st_out(ptx::U32x8* p, const ptx::U32x8& v) { ptx::st_stream_v8(p, v); }
__device__ __forceinline__ uint32_t triad1(uint32_t b, uint32_t c, float s) {
  return __float_as_uint(fmaf(s, __uint_as_float(c), __uint_as_float(b)));
}
__device__ __forceinline__ uint4 triad_vec(const uint4& b, const uint4& c, float s) {
  return make_uint4(triad1(b.x, c.x, s), triad1(b.y, c.y, s), triad1(b.z, c.z, s), triad1(b.w, c.w, s));
}
__device__ __forceinline__ ptx::U32x8 triad_vec(const ptx::U32x8& b, const ptx::U32x8& c, float s) {
  ptx::U32x8 r;
#pragma unroll
  for (int k = 0; k < 8; ++k) r.v[k] = triad1(b.v[k], c.v[k], s);
  return r;
}

template <typename V, int U, bool kPut>
__global__ void __launch_bounds__(512)
    triad_put_ldst_kernel(V* __restrict__ a_local, V* __restrict__ a_peer, const V* __restrict__ b,
                          const V* __restrict__ c, float s, size_t nvec, int blocked, SyncOps sync,
                          const uint32_t* arrive_flag, uint32_t arrive_epoch) {
  if (!cta_prologue_wait(sync)) return;
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
    V vb[U], vc[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      vb[k] = ld_in(b + i + k * stride);
      vc[k] = ld_in(c + i + k * stride);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const V va = triad_vec(vb[k], vc[k], s);
      if (kPut) st_out(a_peer + i + k * stride, va);
      st_out(a_local + i + k * stride, va);
    }
  }
  for (; i < end; i += stride) {
    const V va = triad_vec(ld_in(b + i), ld_in(c + i), s);
    if (kPut) st_out(a_peer + i, va);
    st_out(a_local + i, va);
  }
  cta_epilogue(sync, arrive_flag, arrive_epoch);
}

// Halo mode of the LdSt engine: triad over `ratio` * n_put_vec vectors, the first n_put_vec of them
// (the halo) are also stored into the peer.  Work is dealt in 16 KiB tiles, one halo tile followed by
// ratio-1 interior tiles, so NVLink-bound and HBM-bound tiles interleave inside every CTA.
constexpr int kHaloTileVec = 1024;  // uint4 per tile = 16 KiB
template <bool kPut>
__global__ void __launch_bounds__(512)
    triad_halo_ldst_kernel(uint4* __restrict__ a_local, uint4* __restrict__ a_peer,
                           const uint4* __restrict__ b, const uint4* __restrict__ c, float s,
                           size_t n_put_vec, int ratio, SyncOps sync, const uint32_t* arrive_flag,
                           uint32_t arrive_epoch) {
  if (!cta_prologue_wait(sync)) return;
  const size_t halo_tiles = n_put_vec / kHaloTileVec;
  const size_t total_tiles = halo_tiles * ratio;
  for (size_t t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const size_t g = t / ratio, r = t % ratio;
    const bool halo = r == 0;
    const size_t base = (halo ? g : halo_tiles + (ratio - 1) * g + (r - 1)) * kHaloTileVec;
#pragma unroll
    for (int v0 = 0; v0 < kHaloTileVec; v0 += 1024) {
      uint4 vb[2], vc[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        vb[k] = ld_in(b + base + v0 + threadIdx.x + k * 512);
        vc[k] = ld_in(c + base + v0 + threadIdx.x + k * 512);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint4 va = triad_vec(vb[k], vc[k], s);
        if (kPut && halo) st_out(a_peer + base + v0 + threadIdx.x + k * 512, va);
        st_out(a_local + base + v0 + threadIdx.x + k * 512, va);
      }
    }
  }
  cta_epilogue(sync, arrive_flag, arrive_epoch);
}

// ------------------------------------------------------------- TMA engine ----
constexpr int kMathWarps = 4;
constexpr int kTmaThreads = 32 * (1 + kMathWarps);

// Dynamic smem: [stages][2][tile_bytes] (b tile, c tile) | full[stages] | computed[stages]
// kHint (EXPERIMENTAL, opt-in): L2 evict_first policy on the streamed bulk loads and the local bulk store.
template <bool kPut, bool kHint = false>
__global__ void __launch_bounds__(kTmaThreads)
    triad_put_tma_kernel(float* __restrict__ a_local, float* __restrict__ a_peer,
                         const float* __restrict__ b, const float* __restrict__ c, float s,
                         size_t n_bytes /*multiple of 16*/, uint32_t tile_bytes, int stages,
                         size_t put_bytes /*halo: multiple of tile_bytes; == n_bytes when ratio == 1*/,
                         int ratio /*n_bytes == ratio * put_bytes*/,
                         int halo_ctas /*EXPERIMENTAL: > 0 dedicates CTAs [0,halo_ctas) to the halo*/,
                         SyncOps sync, const uint32_t* arrive_flag, uint32_t arrive_epoch) {
  extern __shared__ __align__(128) unsigned char smem[];
  const size_t stage_stride = 2 * static_cast<size_t>(tile_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + stages * stage_stride);
  uint64_t* computed = full + stages;

  if (!cta_prologue_wait(sync)) return;

  if (threadIdx.x == 0) {
    for (int st = 0; st < stages; ++st) {
      ptx::mbar_init(&full[st], 1);
      ptx::mbar_init(&computed[st], kMathWarps);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  const size_t tiles_total = (n_bytes + tile_bytes - 1) / tile_bytes;
  // Split scheduling (experimental, halo mode only): CTAs [0, halo_ctas) stream the halo tiles (the
  // NVLink-bound work), the remaining CTAs stream the interior (HBM-bound), so neither stream queues
  // behind the other inside a CTA's in-order DMA thread.
  const bool split = ratio > 1 && halo_ctas > 0 && halo_ctas < static_cast<int>(gridDim.x);
  const bool halo_cta = split && static_cast<int>(blockIdx.x) < halo_ctas;
  const size_t split_idx = halo_cta ? blockIdx.x : blockIdx.x - halo_ctas;
  const size_t split_stride = halo_cta ? halo_ctas : gridDim.x - halo_ctas;
  const size_t split_tiles = halo_cta ? put_bytes / tile_bytes : (n_bytes - put_bytes) / tile_bytes;
  const size_t n = split ? (split_tiles > split_idx ? (split_tiles - split_idx + split_stride - 1) / split_stride : 0)
                         : (tiles_total > blockIdx.x ? (tiles_total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0);
  // Halo mode (ratio R > 1): the triad runs over R * put_bytes but only the first put_bytes (the
  // halo) travel to the peer.  Logical tiles interleave one halo tile with R-1 interior tiles, so
  // the NVLink stream and the HBM-only stream of every CTA advance together instead of one after
  // the other (the reference's autotuner balances command durations the same way).
  auto tile_off = [&](size_t j) {
    if (split) return (halo_cta ? 0 : put_bytes) + (split_idx + j * split_stride) * tile_bytes;
    const size_t t = static_cast<size_t>(blockIdx.x) + j * gridDim.x;
    if (ratio <= 1) return t * tile_bytes;
    const size_t g = t / ratio, r = t % ratio;
    return r == 0 ? g * tile_bytes : put_bytes + ((ratio - 1) * g + (r - 1)) * tile_bytes;
  };
  auto tile_is_halo = [&](size_t j) {
    if (split) return halo_cta;
    return ratio <= 1 || (static_cast<size_t>(blockIdx.x) + j * gridDim.x) % ratio == 0;
  };
  auto tile_len = [&](size_t j) {
    const size_t off = tile_off(j);
    return static_cast<uint32_t>(n_bytes - off < tile_bytes ? n_bytes - off : tile_bytes);
  };
  const unsigned char* bb = reinterpret_cast<const unsigned char*>(b);
  const unsigned char* cb = reinterpret_cast<const unsigned char*>(c);
  unsigned char* alb = reinterpret_cast<unsigned char*>(a_local);
  unsigned char* apb = reinterpret_cast<unsigned char*>(a_peer);

  const int warp = threadIdx.x >> 5;
  if (warp == 0) {
    if (threadIdx.x == 0) {
      const uint64_t policy = kHint ? ptx::l2_policy_evict_first() : 0;
      auto issue_load = [&](size_t j) {
        const int st = static_cast<int>(j % stages);
        const uint32_t len = tile_len(j);
        unsigned char* sb = smem + st * stage_stride;
        ptx::mbar_arrive_expect_tx(&full[st], 2 * len);
        if (kHint) {
          ptx::bulk_g2s_hint(sb, bb + tile_off(j), len, &full[st], policy);
          ptx::bulk_g2s_hint(sb + tile_bytes, cb + tile_off(j), len, &full[st], policy);
        } else {
          ptx::bulk_g2s(sb, bb + tile_off(j), len, &full[st]);
          ptx::bulk_g2s(sb + tile_bytes, cb + tile_off(j), len, &full[st]);
        }
      };
      const size_t lookahead = static_cast<size_t>(stages - 1);
      for (size_t j = 0; j < lookahead && j < n; ++j) issue_load(j);
      for (size_t j = 0; j < n; ++j) {
        const int st = static_cast<int>(j % stages);
        ptx::mbar_wait(&computed[st], static_cast<uint32_t>((j / stages) & 1));
        const unsigned char* sa = smem + st * stage_stride;  // `a` overwrote the b tile
        if (kHint)
          ptx::bulk_s2g_hint(alb + tile_off(j), sa, tile_len(j), policy);
        else
          ptx::bulk_s2g(alb + tile_off(j), sa, tile_len(j));
        if (kPut && tile_is_halo(j)) ptx::bulk_s2g(apb + tile_off(j), sa, tile_len(j));
        ptx::bulk_commit();
        const size_t nxt = j + lookahead;
        if (nxt < n) {
          ptx::bulk_wait_read<1>();
          issue_load(nxt);
        }
      }
      ptx::bulk_wait<0>();
      asm volatile("fence.proxy.async;" ::: "memory");
    }
  } else {
    const int mt = threadIdx.x - 32;  // 0 .. 32*kMathWarps-1
    for (size_t j = 0; j < n; ++j) {
      const int st = static_cast<int>(j % stages);
      ptx::mbar_wait(&full[st], static_cast<uint32_t>((j / stages) & 1));
      float4* sb = reinterpret_cast<float4*>(smem + st * stage_stride);
      const float4* sc = reinterpret_cast<const float4*>(smem + st * stage_stride + tile_bytes);
      const uint32_t nv = tile_len(j) / 16;
      for (uint32_t v = mt; v < nv; v += 32 * kMathWarps) sb[v] = triad4(sb[v], sc[v], s);
      ptx::fence_proxy_async_smem();  // generic-proxy smem writes -> visible to TMA store
      __syncwarp();
      if ((threadIdx.x & 31) == 0) ptx::mbar_arrive(&computed[st]);
    }
  }
  cta_epilogue(sync, arrive_flag, arrive_epoch);
}

// ---------------------------------------------------- inputs and checking ----
// b and c of rank r at element i (payload.h): integers in [0, 1023] and [0, 7] drawn from one hash of (i, r).
__global__ void fill_triad_kernel(float* __restrict__ b, float* __restrict__ c, size_t n,
                                  int rank) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t w = triad_word(i, rank);
    b[i] = static_cast<float>(triad_b_bits(w));
    c[i] = static_cast<float>(triad_c_bits(w));
  }
}

__global__ void verify_triad_kernel(const float* __restrict__ a, size_t n, int src_rank, float s,
                                    unsigned long long* mismatch_count) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t w = triad_word(i, src_rank);
    const float want = fmaf(s, static_cast<float>(triad_c_bits(w)), static_cast<float>(triad_b_bits(w)));
    bad += (__ldcg(a + i) != want);
  }
  for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(mismatch_count, bad);
}

}  // namespace

int launch_triad_put(const TriadPutArgs& args, CopyEngine engine, const CopyTuning& tune,
                     const SyncOps& sync, const uint32_t* arrive_flag, uint32_t arrive_epoch,
                     int device, cudaStream_t stream) {
  HPCP_REQUIRE(args.n > 0, "triad_put: n must be positive (an empty triad launches nothing)");
  HPCP_REQUIRE(args.n % 4 == 0, "triad_put: n must be a multiple of 4 elements");
  // Every engine moves 16-byte vectors (LDG/STG.128 or cp.async.bulk); a_peer only matters when there is a put.
  HPCP_REQUIRE(((reinterpret_cast<uintptr_t>(args.a_local) | reinterpret_cast<uintptr_t>(args.a_peer) |
                 reinterpret_cast<uintptr_t>(args.b) | reinterpret_cast<uintptr_t>(args.c)) & 15) == 0,
               "triad_put: pointers must be 16-byte aligned");
  const size_t n_put = args.n_put == 0 ? args.n : args.n_put;
  HPCP_REQUIRE(n_put <= args.n && args.n % n_put == 0, "triad_put: n must be a multiple of n_put");
  const int ratio = static_cast<int>(args.n / n_put);
  HPCP_REQUIRE(sync.signal_flag == nullptr || sync.ticket != nullptr,
               "triad_put: a signal needs a ticket counter");
  // Every refusal comes before the first CUDA call (device_sm_count), so a bad call never reaches the device.
  const size_t nvec = args.n / 4;
  const bool put = args.a_peer != nullptr;
  int ctas = 0;
  if (engine == CopyEngine::kLdSt && ratio > 1) {
    HPCP_REQUIRE((n_put / 4) % kHaloTileVec == 0, "triad_put: halo (n_put) must be a multiple of 16 KiB");
    const size_t tiles = (n_put / 4 / kHaloTileVec) * static_cast<size_t>(ratio);
    const int cap = tune.ctas > 0 ? tune.ctas : device_sm_count(device) * 2;
    ctas = static_cast<int>(std::min<size_t>(tiles, static_cast<size_t>(cap)));
    uint4* al = reinterpret_cast<uint4*>(args.a_local);
    uint4* ap = reinterpret_cast<uint4*>(args.a_peer);
    const uint4* b = reinterpret_cast<const uint4*>(args.b);
    const uint4* c = reinterpret_cast<const uint4*>(args.c);
    if (put)
      triad_halo_ldst_kernel<true><<<ctas, 512, 0, stream>>>(al, ap, b, c, args.s, n_put / 4, ratio, sync,
                                                             arrive_flag, arrive_epoch);
    else
      triad_halo_ldst_kernel<false><<<ctas, 512, 0, stream>>>(al, ap, b, c, args.s, n_put / 4, ratio, sync,
                                                              arrive_flag, arrive_epoch);
  } else if (engine == CopyEngine::kLdSt) {
    const int threads = tune.threads > 0 ? std::min(tune.threads, 512) : 512;
    const int unroll = tune.unroll > 0 ? tune.unroll : 2;
    const size_t per_cta = static_cast<size_t>(threads) * unroll * (tune.vec_bytes == 32 ? 2 : 1);
    const size_t want = std::max<size_t>(1, (nvec + per_cta - 1) / per_cta);
    const int cap = tune.ctas > 0 ? tune.ctas : device_sm_count(device) * 2;
    ctas = static_cast<int>(std::min<size_t>(want, static_cast<size_t>(cap)));
    const bool wide = tune.vec_bytes == 32 && args.n % 8 == 0 &&
                      ((reinterpret_cast<uintptr_t>(args.a_local) | reinterpret_cast<uintptr_t>(args.a_peer) |
                        reinterpret_cast<uintptr_t>(args.b) | reinterpret_cast<uintptr_t>(args.c)) & 31) == 0;
#define HPCP_TRIAD_LAUNCH(V, U)                                                                      \
  do {                                                                                               \
    V* al = reinterpret_cast<V*>(args.a_local);                                                      \
    V* ap = reinterpret_cast<V*>(args.a_peer);                                                       \
    const V* b = reinterpret_cast<const V*>(args.b);                                                 \
    const V* c = reinterpret_cast<const V*>(args.c);                                                 \
    const size_t nv = args.n * sizeof(float) / sizeof(V);                                            \
    if (put)                                                                                         \
      triad_put_ldst_kernel<V, U, true><<<ctas, threads, 0, stream>>>(                               \
          al, ap, b, c, args.s, nv, tune.blocked, sync, arrive_flag, arrive_epoch);                  \
    else                                                                                             \
      triad_put_ldst_kernel<V, U, false><<<ctas, threads, 0, stream>>>(                              \
          al, ap, b, c, args.s, nv, tune.blocked, sync, arrive_flag, arrive_epoch);                  \
  } while (0)
    if (wide) {
      switch (unroll) {
        case 1: HPCP_TRIAD_LAUNCH(ptx::U32x8, 1); break;
        default: HPCP_TRIAD_LAUNCH(ptx::U32x8, 2); break;
      }
    } else {
      switch (unroll) {
        case 1: HPCP_TRIAD_LAUNCH(uint4, 1); break;
        case 4: HPCP_TRIAD_LAUNCH(uint4, 4); break;
        default: HPCP_TRIAD_LAUNCH(uint4, 2); break;
      }
    }
#undef HPCP_TRIAD_LAUNCH
  } else {
    const uint32_t tile_bytes = static_cast<uint32_t>((tune.stage_kb > 0 ? tune.stage_kb : 16) * 1024);
    const int stages = tune.stages > 0 ? tune.stages : 6;
    HPCP_REQUIRE(stages >= 2, "triad_put: TMA engine needs >= 2 stages");
    const size_t smem = static_cast<size_t>(stages) * 2 * tile_bytes + static_cast<size_t>(stages) * 16;
    HPCP_REQUIRE(smem <= 227 * 1024, "triad_put: TMA stages exceed 227 KiB of shared memory");
    const size_t n_bytes = args.n * sizeof(float);
    const size_t put_bytes = n_put * sizeof(float);
    HPCP_REQUIRE(ratio == 1 || put_bytes % tile_bytes == 0,
                 "triad_put: halo (n_put) must be a multiple of the TMA tile size");
    const size_t tiles = std::max<size_t>(1, (n_bytes + tile_bytes - 1) / tile_bytes);
    const int per_sm = std::max(1, static_cast<int>((227 * 1024) / smem));
    const int cap = tune.ctas > 0 ? tune.ctas : device_sm_count(device) * per_sm;
    ctas = static_cast<int>(std::min<size_t>(tiles, static_cast<size_t>(cap)));
    if (tune.l2_hint != 0) {  // experimental variant with L2 cache-policy operands
      if (put) {
        HPCP_ENABLE_SMEM((triad_put_tma_kernel<true, true>), smem);
        triad_put_tma_kernel<true, true><<<ctas, kTmaThreads, smem, stream>>>(
            args.a_local, args.a_peer, args.b, args.c, args.s, n_bytes, tile_bytes, stages, put_bytes, ratio,
            tune.halo_ctas, sync, arrive_flag, arrive_epoch);
      } else {
        HPCP_ENABLE_SMEM((triad_put_tma_kernel<false, true>), smem);
        triad_put_tma_kernel<false, true><<<ctas, kTmaThreads, smem, stream>>>(
            args.a_local, args.a_peer, args.b, args.c, args.s, n_bytes, tile_bytes, stages, put_bytes, ratio,
            tune.halo_ctas, sync, arrive_flag, arrive_epoch);
      }
    } else if (put) {
      HPCP_ENABLE_SMEM(triad_put_tma_kernel<true>, smem);
      triad_put_tma_kernel<true><<<ctas, kTmaThreads, smem, stream>>>(
          args.a_local, args.a_peer, args.b, args.c, args.s, n_bytes, tile_bytes, stages, put_bytes, ratio,
          tune.halo_ctas, sync, arrive_flag, arrive_epoch);
    } else {
      HPCP_ENABLE_SMEM(triad_put_tma_kernel<false>, smem);
      triad_put_tma_kernel<false><<<ctas, kTmaThreads, smem, stream>>>(
          args.a_local, args.a_peer, args.b, args.c, args.s, n_bytes, tile_bytes, stages, put_bytes, ratio,
          tune.halo_ctas, sync, arrive_flag, arrive_epoch);
    }
  }
  HPCP_CUDA(cudaGetLastError());
  return ctas;
}

void launch_fill_triad_inputs(float* b, float* c, size_t n, int rank, cudaStream_t stream) {
  const int threads = 256;
  const int ctas = static_cast<int>(std::min<size_t>((n + threads - 1) / threads, 132 * 8));
  fill_triad_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(b, c, n, rank);
  HPCP_CUDA(cudaGetLastError());
}

void launch_verify_triad(const float* a, size_t n, int src_rank, float s,
                         unsigned long long* mismatch_count, cudaStream_t stream) {
  const int threads = 256;
  const int ctas = static_cast<int>(std::min<size_t>((n + threads - 1) / threads, 132 * 8));
  verify_triad_kernel<<<std::max(ctas, 1), threads, 0, stream>>>(a, n, src_rank, s,
                                                                mismatch_count);
  HPCP_CUDA(cudaGetLastError());
}

}  // namespace hpcp
