// Device enumeration and the per-rank device subset for the miniapps.
//
// Capability parity with aurora.mpich.miniapps/src/include/devices.hpp:22-59:
// if there are fewer devices than ranks every rank gets ONE device chosen
// round-robin (oversubscription); otherwise the devices are dealt in contiguous
// blocks of ndev/size per rank.  PVC "fission" into tiles has no H100
// equivalent (one H100 is one CUDA device; MIG is out of scope), so the
// `fission` switch is accepted and ignored.
#pragma once

#include <cuda_runtime.h>

#include <string>
#include <vector>

namespace hpcp {

inline int visible_device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return n;
}

// Pure function (unit-testable): which ordinals does `rank` of `size` own?
inline std::vector<int> device_subset(int rank, int size, int n_devices) {
  std::vector<int> out;
  if (n_devices <= 0 || size <= 0 || rank < 0) return out;
  if (n_devices < size) {
    out.push_back(rank % n_devices);
    return out;
  }
  const int per_rank = n_devices / size;
  for (int k = 0; k < per_rank; ++k) out.push_back(rank * per_rank + k);
  return out;
}

inline std::vector<int> get_devices(int rank, int size, bool /*fission*/ = false) {
  return device_subset(rank, size, visible_device_count());
}

// The device a rank computes on: the reference indexes its subset with
// rank % subset_size (allreduce-mpi-sycl.cpp:147).
inline int primary_device(int rank, int size, int n_devices) {
  const std::vector<int> mine = device_subset(rank, size, n_devices);
  if (mine.empty()) return -1;
  return mine[static_cast<size_t>(rank) % mine.size()];
}

}  // namespace hpcp
