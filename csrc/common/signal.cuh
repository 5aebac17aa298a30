// Cross-GPU signalling protocol (device side).
//
// Every rank owns a "signal pad": an array of 32-bit words that lives in
// peer-mapped memory so that any GPU can store into it over NVLink.  Words are
// *monotonic epochs*: a writer publishes `epoch` with st.release.sys after its
// data stores, a reader spins with ld.acquire.sys until word >= epoch.  Pads are
// never reset between iterations, so there is no reset race.
//
// This replaces the reference's synchronisation calls:
//   MPI_Win_fence      p2p/peer2pear.cpp:76-81      -> put + signal / wait
//   MPI_Waitall        p2p/peer2pear.cpp:44         -> wait on the done word
//   MPI_Barrier        p2p/peer2pear.cpp:26         -> barrier_all()
//   blocking Send/Recv allreduce-mpi-sycl.cpp:50-58 -> per-chunk arrival words
//
// A hung peer must produce an error, not a hang ("failure
// detection"): every spin has a %globaltimer deadline; on expiry the waiter
// records a code in a status word and returns false so the kernel can drain.
#pragma once

#include "ptx.cuh"
#include "signal_layout.h"

namespace hpcp {

__device__ __forceinline__ bool epoch_reached(uint32_t seen, uint32_t want) {
  return static_cast<int32_t>(seen - want) >= 0;
}

// Spin until *flag >= want (wrap-safe).  One thread calls this.
__device__ __forceinline__ bool wait_epoch(const uint32_t* flag, uint32_t want,
                                           uint64_t timeout_ns, uint32_t* status) {
  if (epoch_reached(ptx::ld_acquire_sys(flag), want)) return true;
  const uint64_t t0 = ptx::globaltimer_ns();
  unsigned spins = 0;
  while (true) {
    if (epoch_reached(ptx::ld_acquire_sys(flag), want)) return true;
    if ((++spins & 0x3ff) == 0) {
      if (status != nullptr && ptx::ld_relaxed_sys(status) != kStatusOk) return false;
      if (timeout_ns != 0 && ptx::globaltimer_ns() - t0 > timeout_ns) {
        if (status != nullptr) ptx::st_relaxed_sys(status, kStatusTimeout);
        return false;
      }
    }
  }
}

// Publish after this CTA's data stores.  Call from ONE thread after a
// __syncthreads(): the barrier orders the CTA's stores before this thread, the
// system fence + release store make them visible to the peer before the word.
__device__ __forceinline__ void publish_epoch(uint32_t* flag_on_peer, uint32_t epoch) {
  ptx::fence_acq_rel_sys();
  ptx::st_release_sys(flag_on_peer, epoch);
}

// Same, without the stand-alone fence: st.release.sys is itself cumulative over
// everything that happens-before it (the CTA's stores, ordered by the preceding
// bar.sync), so hot per-chunk publishes pay one system-scope drain instead of two.
__device__ __forceinline__ void publish_epoch_light(uint32_t* flag_on_peer, uint32_t epoch) {
  ptx::st_release_sys(flag_on_peer, epoch);
}

// Grid-wide "last CTA publishes" helper: every CTA calls it (all threads); the
// CTA that takes the final ticket publishes `epoch` to `flag_on_peer`.
// `ticket` is a rank-local counter that counts up forever (no reset):
// launch number L with G CTAs owns tickets [L*G, (L+1)*G).
__device__ __forceinline__ bool last_cta_publish(uint32_t* ticket, uint32_t tickets_target,
                                                 uint32_t* flag_on_peer, uint32_t epoch) {
  __syncthreads();
  bool last = false;
  if (threadIdx.x == 0) {
    ptx::fence_acq_rel_sys();
    const uint32_t t = ptx::atom_acq_rel_gpu_add(ticket, 1u);
    last = (t + 1u == tickets_target);
    if (last) {
      ptx::fence_acq_rel_sys();
      if (flag_on_peer != nullptr) ptx::st_release_sys(flag_on_peer, epoch);
    }
  }
  return last;  // only meaningful on thread 0
}

}  // namespace hpcp
