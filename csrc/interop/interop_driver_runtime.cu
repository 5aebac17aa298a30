// interop (native handles): the same demo through *native* handles.
//
// Reference: sycl_omp_ze_interopt/interop_omp_ze_sycl.cpp:81-116 — ze_driver / ze_context /
// ze_device handles are pulled out of the OpenMP interop object and wrapped into SYCL
// objects with ownership "keep", devices sharing a ze_context grouped into one SYCL context.
// CUDA/H100 analogue: the driver-API objects underneath the runtime — CUdevice, the primary
// CUcontext, the CUstream behind a cudaStream_t, CUdeviceptr behind a void* — are taken from
// the runtime side and used by a driver-API component (and back), via the cached table in
// device_table.h.  No context is ever created or destroyed here: the primary context is
// retained ("keep") because the runtime / PyTorch own it.
#include <cstdio>
#include <iostream>
#include <vector>

#include "../common/cuda_check.h"
#include "../common/driver_api.h"
#include "../kernels/api.h"
#include "device_table.h"

__global__ void write_value(int* p, int n, int value) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = value;
}

int main() {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  using namespace hpcp;
  try {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
      std::cerr << "interop: no CUDA device" << std::endl;
      return 1;
    }
    const DriverApi& d = DriverApi::get();
    const int D = ndev - 1;
    const DeviceNativeInfo& info = xcuda_get_device_info(D);
    HPCP_CUDA(cudaSetDevice(D));
    const int N = 100;

    // The runtime's stream IS a driver stream: same handle, same (primary) context.
    cudaStream_t rt_stream;
    HPCP_CUDA(cudaStreamCreateWithFlags(&rt_stream, cudaStreamNonBlocking));
    CUstream cu_stream = reinterpret_cast<CUstream>(rt_stream);
    CUcontext stream_ctx = nullptr;
    CUgreenCtx green = nullptr;  // 12.5+ ABI of cuStreamGetCtx also reports a green context
    HPCP_CU(d.cuStreamGetCtx(cu_stream, &stream_ctx, &green));
    CUcontext current = nullptr;
    HPCP_CU(d.cuCtxGetCurrent(&current));
    HPCP_REQUIRE(stream_ctx == info.cu_context && current == info.cu_context,
                 "runtime stream / current context is not the primary context from the table");
    std::cout << "Device " << D << ": CUdevice=" << info.cu_device << " primary CUcontext shared by runtime "
              << "and driver API; P2P group size " << info.peers.size() + 1 << std::endl;

    std::cout << "Driver -> Runtime" << std::endl;
    CUdeviceptr drv_mem = 0;
    HPCP_CU(d.cuMemAlloc(&drv_mem, N * sizeof(int)));
    write_value<<<1, 128, 0, rt_stream>>>(reinterpret_cast<int*>(drv_mem), N, N);  // runtime kernel, driver memory
    HPCP_CUDA(cudaGetLastError());
    std::cout << "   Runtime memcpy using the driver pointer" << std::endl;
    std::vector<int> host(N, -1);
    HPCP_CUDA(cudaMemcpyAsync(host.data(), reinterpret_cast<void*>(drv_mem), N * sizeof(int),
                              cudaMemcpyDeviceToHost, rt_stream));
    HPCP_CUDA(cudaStreamSynchronize(rt_stream));
    for (int i = 0; i < N; ++i) HPCP_REQUIRE(host[i] == N, "driver -> runtime data mismatch");

    std::cout << "Runtime -> Driver" << std::endl;
    int* rt_mem = nullptr;
    HPCP_CUDA(cudaMalloc(&rt_mem, N * sizeof(int)));
    launch_fill_pattern(reinterpret_cast<uint32_t*>(rt_mem), N, 7u, rt_stream);
    std::cout << "  Driver memcpy using the runtime pointer, on the runtime's stream" << std::endl;
    HPCP_CU(d.cuMemcpyDtoDAsync(drv_mem, reinterpret_cast<CUdeviceptr>(rt_mem), N * sizeof(int), cu_stream));
    std::vector<int> a(N), b(N);
    HPCP_CUDA(cudaMemcpyAsync(a.data(), rt_mem, N * sizeof(int), cudaMemcpyDeviceToHost, rt_stream));
    HPCP_CUDA(cudaMemcpyAsync(b.data(), reinterpret_cast<void*>(drv_mem), N * sizeof(int),
                              cudaMemcpyDeviceToHost, rt_stream));
    HPCP_CUDA(cudaStreamSynchronize(rt_stream));
    for (int i = 0; i < N; ++i) HPCP_REQUIRE(a[i] == b[i], "runtime -> driver data mismatch");

    HPCP_CU(d.cuMemFree(drv_mem));
    HPCP_CUDA(cudaFree(rt_mem));
    HPCP_CUDA(cudaStreamDestroy(rt_stream));
    std::cout << "Computation Done" << std::endl;
    return 0;
  } catch (const std::exception& e) {
    std::cerr << "interop: ERROR: " << e.what() << std::endl;
    return 1;
  }
}
