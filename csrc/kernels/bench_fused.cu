// K-fused-bench: the concurrency benchmark's command group as ONE persistent kernel.
//
// The reference submits each command (compute kernel `C`, copies `X2Y`)
// separately and measures whether the runtime overlaps them
// (concurency/bench_sycl.cpp:84-121; four idioms in concurency/README.md:51-101).
// `fused` mode removes the runtime from the question: the grid is partitioned
// between the commands of the group —
//   busy  CTAs : the dependent-FMA chain of `C`        (bench.hpp:23-31 maths)
//   triad CTAs : a = b + s*c stream tile of `A`
//   copy  CTAs : one elected DMA thread per CTA streams the copy through smem
//                with cp.async.bulk (TMA); src/dst may be local HBM, a peer GPU
//                (NVLink), pinned host memory (PCIe, zero-copy) or managed memory
// — so compute and data movement are co-resident on the SMs for the whole launch.
#include "api.h"

#include <algorithm>

#include "../common/cuda_check.h"
#include "../common/ptx.cuh"
#include "../concurency/bench.hpp"

namespace hpcp {

namespace {

struct FusedSlot {
  int kind;
  int cta_begin;
  int cta_end;
  size_t n;
  size_t tripcount;
  void* dst;
  const void* src;
  float* a;
  const float* b;
  const float* c;
  float s;
};

struct FusedTable {
  int n;
  FusedSlot slot[kFusedMaxCommands];
};

__device__ __forceinline__ void cta_copy_tma(unsigned char* smem, unsigned char* dst,
                                             const unsigned char* src, size_t bytes16, int lcta,
                                             int ncta, uint32_t stage_bytes, int stages) {
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + static_cast<size_t>(stages) * stage_bytes);
  if (threadIdx.x != 0) return;
  for (int s = 0; s < stages; ++s) ptx::mbar_init(&full[s], 1);
  ptx::fence_mbar_init();
  const size_t tiles_total = (bytes16 + stage_bytes - 1) / stage_bytes;
  const size_t n = tiles_total > static_cast<size_t>(lcta)
                       ? (tiles_total - lcta + ncta - 1) / ncta
                       : 0;
  auto tile_off = [&](size_t j) { return (static_cast<size_t>(lcta) + j * ncta) * stage_bytes; };
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
      ptx::bulk_wait_read<1>();
      issue_load(nxt);
    }
  }
  ptx::bulk_wait<0>();
}

__device__ __forceinline__ void cta_copy_ldst(uint4* dst, const uint4* src, size_t nvec, int lcta,
                                              int ncta) {
  const size_t stride = static_cast<size_t>(ncta) * blockDim.x;
  size_t i = static_cast<size_t>(lcta) * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = ptx::ld_weak_v4(src + i + k * stride);
#pragma unroll
    for (int k = 0; k < 4; ++k) ptx::st_stream_v4(dst + i + k * stride, v[k]);
  }
  for (; i < nvec; i += stride) ptx::st_stream_v4(dst + i, ptx::ld_weak_v4(src + i));
}

__global__ void __launch_bounds__(512)
    fused_bench_kernel(const __grid_constant__ FusedTable table, int use_tma, uint32_t stage_bytes,
                       int stages) {
  extern __shared__ __align__(128) unsigned char smem[];
  int which = 0;
  for (int k = 0; k < table.n; ++k)
    if (static_cast<int>(blockIdx.x) >= table.slot[k].cta_begin &&
        static_cast<int>(blockIdx.x) < table.slot[k].cta_end)
      which = k;
  const FusedSlot& me = table.slot[which];
  const int lcta = static_cast<int>(blockIdx.x) - me.cta_begin;
  const int ncta = me.cta_end - me.cta_begin;

  if (me.kind == static_cast<int>(FusedKind::kBusy)) {
    const size_t stride = static_cast<size_t>(ncta) * blockDim.x;
    for (size_t j = static_cast<size_t>(lcta) * blockDim.x + threadIdx.x; j < me.n; j += stride)
      me.a[j] = con::busy_wait<float>(me.tripcount, static_cast<float>(j));
  } else if (me.kind == static_cast<int>(FusedKind::kTriad)) {
    const size_t nvec = me.n / 4;
    const float4* b = reinterpret_cast<const float4*>(me.b);
    const float4* c = reinterpret_cast<const float4*>(me.c);
    float4* a = reinterpret_cast<float4*>(me.a);
    const size_t stride = static_cast<size_t>(ncta) * blockDim.x;
    size_t i = static_cast<size_t>(lcta) * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < nvec; i += 4 * stride) {  // 8 independent 128-bit loads in flight
      float4 vb[4], vc[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        vb[k] = __ldcs(b + i + k * stride);
        vc[k] = __ldcs(c + i + k * stride);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        __stcs(a + i + k * stride, make_float4(fmaf(me.s, vc[k].x, vb[k].x), fmaf(me.s, vc[k].y, vb[k].y),
                                               fmaf(me.s, vc[k].z, vb[k].z), fmaf(me.s, vc[k].w, vb[k].w)));
    }
    for (; i < nvec; i += stride) {
      const float4 vb = __ldcs(b + i), vc = __ldcs(c + i);
      __stcs(a + i, make_float4(fmaf(me.s, vc.x, vb.x), fmaf(me.s, vc.y, vb.y),
                                fmaf(me.s, vc.z, vb.z), fmaf(me.s, vc.w, vb.w)));
    }
    if (lcta == 0 && threadIdx.x < (me.n & 3)) {
      const size_t i = (me.n & ~static_cast<size_t>(3)) + threadIdx.x;
      me.a[i] = fmaf(me.s, me.c[i], me.b[i]);
    }
  } else {
    const size_t bytes = me.n * sizeof(float);
    const size_t bytes16 = bytes & ~static_cast<size_t>(15);
    if (use_tma)
      cta_copy_tma(smem, static_cast<unsigned char*>(me.dst),
                   static_cast<const unsigned char*>(me.src), bytes16, lcta, ncta, stage_bytes,
                   stages);
    else
      cta_copy_ldst(static_cast<uint4*>(me.dst), static_cast<const uint4*>(me.src), bytes16 / 16,
                    lcta, ncta);
    if (lcta == 0 && threadIdx.x < (bytes & 15))
      static_cast<unsigned char*>(me.dst)[bytes16 + threadIdx.x] =
          static_cast<const unsigned char*>(me.src)[bytes16 + threadIdx.x];
  }
}

__global__ void busy_wait_kernel(float* __restrict__ out, size_t n, size_t tripcount) {
  const size_t j = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j < n) out[j] = con::busy_wait<float>(tripcount, static_cast<float>(j));
}

}  // namespace

void launch_busy_wait(float* out, size_t n_items, size_t tripcount, cudaStream_t stream) {
  const int threads = static_cast<int>(std::min<size_t>(std::max<size_t>(n_items, 1), 128));
  const unsigned ctas = static_cast<unsigned>((std::max<size_t>(n_items, 1) + threads - 1) / threads);
  // Keep the SM's shared-memory carveout at its maximum even though this kernel uses none: a
  // smem-hungry kernel launched while `C` is running (TMA copies, the wgmma tile loop) must be
  // able to co-reside on the same SM, which is the whole point of the benchmark.
  static const cudaError_t carveout_once = cudaFuncSetAttribute(
      busy_wait_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  (void)carveout_once;
  busy_wait_kernel<<<ctas, threads, 0, stream>>>(out, n_items, tripcount);
  HPCP_CUDA(cudaGetLastError());
}

int launch_fused_bench(const FusedCommand* cmds, int n_cmds, CopyEngine engine,
                       const CopyTuning& tune, int device, cudaStream_t stream) {
  HPCP_REQUIRE(n_cmds >= 1 && n_cmds <= kFusedMaxCommands, "fused bench: 1..8 commands per group");
  const int sms = device_sm_count(device);
  const int threads = 512;

  // CTA budget: busy commands take what their work-item count needs (capped);
  // the rest of one resident wave (one CTA per SM) is shared by triad (weight 4)
  // and copy (weight 1) commands.
  int ctas[kFusedMaxCommands] = {0};
  int fixed = 0, weight_sum = 0;
  for (int k = 0; k < n_cmds; ++k) {
    if (cmds[k].ctas > 0) {
      ctas[k] = cmds[k].ctas;
      fixed += ctas[k];
    } else if (cmds[k].kind == FusedKind::kBusy) {
      const size_t want = (std::max<size_t>(cmds[k].n, 1) + threads - 1) / threads;
      ctas[k] = static_cast<int>(std::min<size_t>(want, static_cast<size_t>(std::max(1, sms / 2))));
      // a busy CTA only needs as many threads as work-items, but the block size is shared
      fixed += ctas[k];
    } else {
      weight_sum += cmds[k].kind == FusedKind::kTriad ? 4 : 1;
    }
  }
  // Two resident CTAs per SM (4 x 16 KiB smem stages each): one wave of 2*SMs CTAs.
  const int pool = std::max(2 * sms - fixed, n_cmds);
  for (int k = 0; k < n_cmds; ++k) {
    if (ctas[k] != 0) continue;
    const int w = cmds[k].kind == FusedKind::kTriad ? 4 : 1;
    ctas[k] = std::max(1, pool * w / std::max(weight_sum, 1));
  }

  FusedTable table{};
  table.n = n_cmds;
  int next = 0;
  for (int k = 0; k < n_cmds; ++k) {
    FusedSlot& s = table.slot[k];
    s.kind = static_cast<int>(cmds[k].kind);
    s.cta_begin = next;
    s.cta_end = next + ctas[k];
    next = s.cta_end;
    s.n = cmds[k].n;
    s.tripcount = cmds[k].tripcount;
    s.dst = cmds[k].dst;
    s.src = cmds[k].src;
    s.a = cmds[k].a;
    s.b = cmds[k].b;
    s.c = cmds[k].c;
    s.s = cmds[k].s;
    if (cmds[k].kind == FusedKind::kCopy)
      HPCP_REQUIRE((reinterpret_cast<uintptr_t>(s.dst) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(s.src) & 15) == 0,
                   "fused bench: copy pointers must be 16-byte aligned");
  }

  const uint32_t stage_bytes = static_cast<uint32_t>((tune.stage_kb > 0 ? tune.stage_kb : 16) * 1024);
  const int stages = tune.stages > 0 ? tune.stages : 4;
  const size_t smem = engine == CopyEngine::kTma
                          ? static_cast<size_t>(stages) * stage_bytes + static_cast<size_t>(stages) * 8
                          : 0;
  HPCP_REQUIRE(smem <= 227 * 1024, "fused bench: TMA stages exceed 227 KiB of shared memory");
  HPCP_ENABLE_SMEM(fused_bench_kernel, smem);
  fused_bench_kernel<<<next, threads, smem, stream>>>(table, engine == CopyEngine::kTma ? 1 : 0,
                                                      stage_bytes, stages);
  HPCP_CUDA(cudaGetLastError());
  return next;
}

}  // namespace hpcp
