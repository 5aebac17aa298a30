// interop (direct): two independently written components share a device, a stream
// and memory without copying handles through any third layer.
//
// Reference: sycl_omp_ze_interopt/interop_omp_sycl.cpp:40-75 — memory allocated and
// written by the OpenMP runtime is read by a SYCL memcpy, and memory allocated by SYCL
// is read by an OpenMP kernel, through `omp interop ... prefer_type("sycl")`.
// CUDA/H100 analogue: a "foreign runtime" component (stream-ordered allocator with its
// own memory pool + its own non-blocking stream + its own kernels, the way an OpenMP
// or PyTorch runtime would own them) and this suite's kernels (csrc/kernels) operate on
// each other's allocations and stream.  The PyTorch flavour of the same demo is
// hpc_patterns_b200/models/interop.py.
#include <cassert>
#include <cstdio>
#include <iostream>
#include <vector>

#include "../common/cuda_check.h"
#include "../common/peer_mem.h"
#include "../kernels/api.h"

namespace foreign {  // stands in for "the other runtime"

__global__ void write_value(int* p, int n, int value) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = value;
}
__global__ void read_into(const int* src, int* dst, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

struct Runtime {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaMemPool_t pool = nullptr;
  explicit Runtime(int dev) : device(dev) {
    HPCP_CUDA(cudaSetDevice(dev));
    HPCP_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    HPCP_CUDA(cudaMemPoolCreate(&pool, &props));
  }
  int* alloc(int n) {
    void* p = nullptr;
    HPCP_CUDA(cudaMallocFromPoolAsync(&p, n * sizeof(int), pool, stream));
    return static_cast<int*>(p);
  }
  void release(int* p) { HPCP_CUDA(cudaFreeAsync(p, stream)); }
  ~Runtime() {
    (void)cudaStreamSynchronize(stream);
    (void)cudaMemPoolDestroy(pool);
    (void)cudaStreamDestroy(stream);
  }
};

}  // namespace foreign

int main() {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  try {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
      std::cerr << "interop: no CUDA device" << std::endl;
      return 1;
    }
    const int D = ndev - 1;  // last device, like the reference picks the last OpenMP device
    const int N = 100;
    foreign::Runtime rt(D);
    std::vector<int> host(N, -1);

    std::cout << "Foreign runtime -> HPCP" << std::endl;
    int* foreign_mem = rt.alloc(N);
    foreign::write_value<<<1, 128, 0, rt.stream>>>(foreign_mem, N, N);
    HPCP_CUDA(cudaGetLastError());
    std::cout << "   HPCP copy kernel using the foreign runtime's pointer and stream" << std::endl;
    int* mine = static_cast<int*>(hpcp::alloc_bytes(N * sizeof(int) + 16, hpcp::AllocKind::kDevice, D, true));
    hpcp::launch_copy(mine, foreign_mem, N * sizeof(int), false, hpcp::CopyEngine::kLdSt, hpcp::CopyTuning{},
                      hpcp::SyncOps{}, D, rt.stream);
    HPCP_CUDA(cudaMemcpyAsync(host.data(), mine, N * sizeof(int), cudaMemcpyDeviceToHost, rt.stream));
    HPCP_CUDA(cudaStreamSynchronize(rt.stream));
    for (int i = 0; i < N; ++i) HPCP_REQUIRE(host[i] == N, "foreign -> HPCP data mismatch");

    std::cout << "HPCP -> Foreign runtime" << std::endl;
    // Do not rely on zero-initialised memory (the reference does, interop_omp_sycl.cpp:71-72):
    // write a known pattern with this suite's fill kernel first.
    hpcp::launch_fill_pattern(reinterpret_cast<uint32_t*>(mine), N, 0x1234u, rt.stream);
    std::cout << "  Foreign kernel reading the HPCP pointer" << std::endl;
    int* foreign_dst = rt.alloc(N);
    foreign::read_into<<<1, 128, 0, rt.stream>>>(mine, foreign_dst, N);
    HPCP_CUDA(cudaGetLastError());
    std::vector<int> a(N), b(N);
    HPCP_CUDA(cudaMemcpyAsync(a.data(), mine, N * sizeof(int), cudaMemcpyDeviceToHost, rt.stream));
    HPCP_CUDA(cudaMemcpyAsync(b.data(), foreign_dst, N * sizeof(int), cudaMemcpyDeviceToHost, rt.stream));
    HPCP_CUDA(cudaStreamSynchronize(rt.stream));
    for (int i = 0; i < N; ++i) HPCP_REQUIRE(a[i] == b[i], "HPCP -> foreign data mismatch");

    rt.release(foreign_mem);
    rt.release(foreign_dst);
    hpcp::free_bytes(mine, hpcp::AllocKind::kDevice);
    std::cout << "Computation Done" << std::endl;
    return 0;
  } catch (const std::exception& e) {
    std::cerr << "interop: ERROR: " << e.what() << std::endl;
    return 1;
  }
}
