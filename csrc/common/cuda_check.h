// Error handling shared by every native component.
//
// The reference aborts through `error()` + MPI_Finalize + exit(1)
// (aurora.mpich.miniapps/src/allreduce/mpi-sycl/allreduce-mpi-sycl.cpp:79-86).
// Here every CUDA runtime / driver failure becomes a C++ exception carrying
// file:line and the CUDA error string, so CLIs can print + exit(1) and the
// Python bindings can surface a RuntimeError instead of killing the process.
#pragma once

#include <cuda_runtime.h>

#include <cstdlib>
#include <sstream>
#include <stdexcept>
#include <string>

namespace hpcp {

struct CudaError : std::runtime_error {
  cudaError_t code;
  CudaError(cudaError_t c, const std::string& what) : std::runtime_error(what), code(c) {}
};

inline void cuda_check(cudaError_t e, const char* expr, const char* file, int line) {
  if (e == cudaSuccess) return;
  std::ostringstream os;
  os << "CUDA error " << static_cast<int>(e) << " (" << cudaGetErrorName(e) << ": "
     << cudaGetErrorString(e) << ") at " << file << ":" << line << " in `" << expr << "`";
  // Clear the sticky-less error so the next call reports its own status.
  (void)cudaGetLastError();
  throw CudaError(e, os.str());
}

[[noreturn]] inline void fail(const std::string& msg, const char* file, int line) {
  std::ostringstream os;
  os << msg << " (" << file << ":" << line << ")";
  throw std::runtime_error(os.str());
}

// Opt a kernel into `bytes` of dynamic shared memory AND ask for the maximum shared-memory
// carveout.  The carveout matters for co-residency: an SM configured for a small carveout by an
// earlier launch cannot host a CTA of a later kernel that needs more until it drains, which
// serialises kernels that were meant to overlap.
template <typename Kernel>
inline void enable_dynamic_smem(Kernel kernel, size_t bytes, const char* file, int line) {
  cuda_check(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(bytes)),
             "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)", file, line);
  cuda_check(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  static_cast<int>(cudaSharedmemCarveoutMaxShared)),
             "cudaFuncSetAttribute(PreferredSharedMemoryCarveout)", file, line);
}

// Call FIRST in main(), before any CUDA call.  CUDA >= 12.2 loads kernels lazily: the first launch of a kernel loads
// its module, and that load cannot complete while another kernel is running on the device.  This suite runs kernels
// that spin on words a peer's kernel will write; when two ranks share a GPU (more ranks than devices) the peer's
// FIRST launch of e.g. `signal_kernel` then waits for the spinning kernel, which waits for that signal: a deadlock
// that only the 30 s device-side deadline breaks (every >= 3-ranks-per-GPU run and the rendezvous / copy-engine
// transports of peer2pear on one GPU would time out).
// Eager loading makes every kernel resident at start-up.  An explicit user setting wins.
inline void prefer_eager_module_loading() { (void)setenv("CUDA_MODULE_LOADING", "EAGER", /*overwrite=*/0); }

}  // namespace hpcp

#define HPCP_ENABLE_SMEM(kernel, bytes) ::hpcp::enable_dynamic_smem((kernel), (bytes), __FILE__, __LINE__)
#define HPCP_CUDA(expr) ::hpcp::cuda_check((expr), #expr, __FILE__, __LINE__)
#define HPCP_FAIL(msg) ::hpcp::fail((msg), __FILE__, __LINE__)
#define HPCP_REQUIRE(cond, msg) \
  do {                          \
    if (!(cond)) HPCP_FAIL(msg); \
  } while (0)
