// Interface between the concurrency driver (host-pure: CLI grammar, autotune,
// verdict — driver.cpp) and the execution backends.
//
// Capability parity with the reference's single `bench<T>()` entry point
// (concurency/bench.hpp:37-40): a backend runs a list of *commands* either one
// after the other ("serial") or concurrently in a backend-specific mode and
// reports the minimum wall time over repetitions, plus per-command minima in
// serial mode.  Differences by design:
//   * backends are runtime objects, so one binary carries the CPU/OpenMP
//     backend and the CUDA backend and the mode is a runtime choice (the
//     reference needs one build per OpenMP mode: run_omp.sh:6-7);
//   * commands: `C` busy-wait FMA chain (identical maths to bench.hpp:23-31),
//     `A` stream triad/axpy tile (HBM-bound compute), `T` wgmma tensor tile,
//     and copies `X2Y` with X,Y in M(alloc) D(evice) H(pinned) S(managed)
//     P(eer GPU over NVLink — new);
//   * byte counts are 64-bit (the reference's `unsigned bytes` overflows at
//     4 GiB, main.cpp:26).
#pragma once

#include <cstddef>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace hpcp {
namespace con {

using Params = std::unordered_map<std::string, size_t>;

struct BenchRequest {
  std::string mode;                   // "serial" or one of Backend::modes()
  std::vector<std::string> commands;  // sanitised tokens: "C", "A", "T", "MD", "DP", ...
  Params params;                      // globalsize_<cmd>, tripcount_C
  bool enable_profiling = false;      // also record device-side (event) times
  int n_queues = -1;                  // -1: backend default for the mode
  int n_repetitions = 10;
  bool verbose = false;
};

// Parameter lookup with a usable error (the API is also reachable from Python with hand-made dicts).
inline size_t require_param(const BenchRequest& req, const std::string& key) {
  const auto it = req.params.find(key);
  if (it == req.params.end())
    throw std::invalid_argument("concurency bench: missing parameter '" + key + "' (commands are sanitised: M2D -> MD)");
  return it->second;
}

struct BenchResult {
  long total_us = 0;                  // min over repetitions of the whole group
  std::vector<long> per_command_us;   // serial mode only: min per command
  std::vector<double> device_us;      // enable_profiling: device-timed per command (may be empty)
  double device_total_us = -1;        // enable_profiling: device-timed span of the group
};

class Backend {
 public:
  virtual ~Backend() = default;
  virtual std::string name() const = 0;
  // Concurrent modes (not including "serial"), e.g. {"in_order","out_of_order"}.
  virtual std::vector<std::string> modes() const = 0;
  // Letters usable as copy endpoints on this backend, e.g. "MDHSP".
  virtual std::string memory_letters() const = 0;
  // Compute commands supported, e.g. "CAT".
  virtual std::string compute_letters() const = 0;
  // Element size of T (float) — all sizes are in elements like the reference.
  virtual BenchResult run(const BenchRequest& req) = 0;
};

// The compute payload: N x 64 dependent FMAs; the data dependence makes the
// duration proportional to N regardless of hardware width, so that two `C`
// commands only overlap if the device truly runs them at the same time.
#if defined(__CUDACC__)
#define HPCP_HD __host__ __device__ __forceinline__
#else
#define HPCP_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define HPCP_PRAGMA_UNROLL _Pragma("unroll")
#else
#define HPCP_PRAGMA_UNROLL
#endif

template <class T>
HPCP_HD T busy_wait(size_t n_iter, T seed) {
  T x = static_cast<T>(1.3f);
  T y = seed;
  for (size_t j = 0; j < n_iter; ++j) {
HPCP_PRAGMA_UNROLL
    for (int k = 0; k < 32; ++k) {
      x = y * x + y;
      y = x * y + x;
    }
  }
  return y;
}

std::unique_ptr<Backend> make_cpu_backend();
// Returns nullptr when the binary was built without CUDA or no GPU is present.
std::unique_ptr<Backend> make_cuda_backend(std::string* why_not);

}  // namespace con
}  // namespace hpcp
