// Inline-PTX vocabulary for sm_90a used by every kernel in this suite.
//
// This is the device-side replacement for the communication calls the
// reference makes through GPU-aware MPICH: system-scope
// acquire/release signal words stand in for MPI_Win_fence / MPI_Waitall /
// MPI_Barrier, vector and TMA-bulk stores to peer-mapped addresses stand in
// for MPI_Put / MPI_Isend, `multimem.*` stands in for MPI_Allreduce.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace hpcp {
namespace ptx {

// ---------------------------------------------------------------- timers ----
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ----------------------------------------------- system-scope signal words ----
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_sys_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_gpu_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_acq_rel_gpu_add(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;"
               : "=r"(old)
               : "l"(p), "r"(v)
               : "memory");
  return old;
}
__device__ __forceinline__ void fence_acq_rel_sys() {
  asm volatile("fence.acq_rel.sys;" ::: "memory");
}
__device__ __forceinline__ void fence_acq_rel_gpu() {
  asm volatile("fence.acq_rel.gpu;" ::: "memory");
}

// --------------------------------------------- 128-bit streaming ld / st ----
// Local HBM source of a put: read-once, keep it out of L1.
__device__ __forceinline__ uint4 ld_stream_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// Peer source of a get.  Peer data may change between launches, so no `.nc`;
// `.relaxed.sys` keeps it coherent with the remote writer without a fence.
__device__ __forceinline__ uint4 ld_peer_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_weak_v4(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream_v4(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// 16-byte floating-point reduction into (peer) memory: REDG.E.ADD.F32x4, performed at the owning GPU's L2.
__device__ __forceinline__ void red_add_f32x4_sys(float* p, const float4& v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// Same for 8 packed bf16 (REDG.E.ADD.BF16x8): half the NVLink bytes, every addition rounds to bf16.
__device__ __forceinline__ void red_add_bf16x8_sys(void* p, const uint4& v) {
  asm volatile("red.relaxed.sys.global.add.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ------------------------------------------------ 32-byte ld / st pairs ----
// 32 bytes per thread as two adjacent 128-bit accesses (sm_90 has no 256-bit LDG/STG): a warp still covers 1 KiB
// contiguous per loop iteration, with twice the bytes in flight per thread of the 16-byte form.
struct alignas(32) U32x8 {
  uint32_t v[8];
};
__device__ __forceinline__ U32x8 ld_stream_v8(const U32x8* p) {
  U32x8 r;
  const uint4 lo = ld_stream_v4(reinterpret_cast<const uint4*>(p));
  const uint4 hi = ld_stream_v4(reinterpret_cast<const uint4*>(p) + 1);
  r.v[0] = lo.x, r.v[1] = lo.y, r.v[2] = lo.z, r.v[3] = lo.w;
  r.v[4] = hi.x, r.v[5] = hi.y, r.v[6] = hi.z, r.v[7] = hi.w;
  return r;
}
__device__ __forceinline__ U32x8 ld_weak_v8(const U32x8* p) {
  U32x8 r;
  const uint4 lo = ld_weak_v4(reinterpret_cast<const uint4*>(p));
  const uint4 hi = ld_weak_v4(reinterpret_cast<const uint4*>(p) + 1);
  r.v[0] = lo.x, r.v[1] = lo.y, r.v[2] = lo.z, r.v[3] = lo.w;
  r.v[4] = hi.x, r.v[5] = hi.y, r.v[6] = hi.z, r.v[7] = hi.w;
  return r;
}
__device__ __forceinline__ void st_stream_v8(U32x8* p, const U32x8& r) {
  st_stream_v4(reinterpret_cast<uint4*>(p), make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]));
  st_stream_v4(reinterpret_cast<uint4*>(p) + 1, make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]));
}

// ------------------------------------------------------------- mbarrier ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Generic-proxy writes to smem -> visible to the async (TMA) proxy.
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ------------------------------------------- TMA bulk (non-tensor) copies ----
// global (local HBM *or* a peer-mapped NVLink address) -> shared, completion on mbarrier.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global (local or peer); completion tracked by bulk async-groups.
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
// Same two copies with an L2 cache-policy operand (createpolicy ... evict_first: streamed once, never re-read).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar,
                                              uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void bulk_s2g_hint(void* gdst, const void* smem_src, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes), "l"(policy)
               : "memory");
}
// shared -> global with an f32 add performed at the destination ("put + accumulate").
__device__ __forceinline__ void bulk_s2g_add_f32(void* gdst, const void* smem_src,
                                                 uint32_t bytes) {
  asm volatile(
      "cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gdst),
      "r"(smem_u32(smem_src)), "r"(bytes)
      : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// Wait until at most N groups still *read* their smem source (smem reusable).
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// Wait until at most N groups are incomplete (writes performed).
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------- NVLS / multimem ----
// In-switch reduction: one load returns the sum over every GPU bound to the
// multicast object (replaces MPI_Allreduce's reduce step).
__device__ __forceinline__ float4 multimem_ld_reduce_add_f32x4(const void* mc_ptr) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
__device__ __forceinline__ int multimem_ld_reduce_add_s32(const void* mc_ptr) {
  int v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.s32 %0, [%1];"
               : "=r"(v)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
// Broadcast store: one store lands in every bound GPU (replaces the allgather step).
__device__ __forceinline__ void multimem_st_f32x4(void* mc_ptr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
// In-switch reduction INTO memory: one 16-byte request, the switch adds it into every bound GPU's copy
// (an all-reduce contribution that leaves the sender once).
__device__ __forceinline__ void multimem_red_add_f32x4(void* mc_ptr, const float4& v) {
  asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void multimem_st_b32(void* mc_ptr, uint32_t v) {
  asm volatile("multimem.st.relaxed.sys.global.b32 [%0], %1;" ::"l"(mc_ptr), "r"(v) : "memory");
}
__device__ __forceinline__ void multimem_red_release_sys_add(void* mc_ptr, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc_ptr), "r"(v)
               : "memory");
}

// ------------------------------------------------------------- helpers ----
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace ptx
}  // namespace hpcp
