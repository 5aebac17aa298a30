// The K-halo field as a definition shared by the kernels (halo_stencil.cu) and their host twin (`halo --cpu`,
// miniapps/halo.cu): the closed-form initial field, the conversions between a field type and its compute type, the
// global-row bound of the verifier, and the dispatch over the field types.  Both sides compile this one copy, so the
// host twin cannot drift from the device.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>
#include <string>

#include "../common/cuda_check.h"
#include "api.h"

namespace hpcp {

// halo_verify_from_init keeps a whole column of the global field in registers: world * rows <= this.
constexpr int kHaloMaxGlobalRows = 128;

// u0(global row, column): a hash folded to [-32, 32) with 10 fractional bits, reproducible on the host
// (models/halo.py::initial_field).  A field of type T starts at u0 rounded to T (exact for float and double).
__host__ __device__ __forceinline__ float halo_u0(uint32_t grow, uint64_t j) {
  const uint32_t jl = static_cast<uint32_t>(j);
  const uint32_t h = (grow * 2654435761u) ^ (jl * 40503u + (jl >> 11));
  return static_cast<float>(static_cast<int>(h & 0xFFFFu) - 32768) * (1.0f / 1024.0f);
}

// Element <-> compute type: widen is exact, narrow rounds to nearest even and keeps subnormals.  The cuda_bf16.h /
// cuda_fp16.h conversions are host functions too, so the host rounds exactly as the kernels do.
template <class T>
struct FieldElem {  // float, double
  using Compute = T;
  __host__ __device__ static __forceinline__ T widen(T x) { return x; }
  __host__ __device__ static __forceinline__ T narrow(T x) { return x; }
};
template <>
struct FieldElem<__nv_bfloat16> {
  using Compute = float;
  __host__ __device__ static __forceinline__ float widen(__nv_bfloat16 x) { return __bfloat162float(x); }
  __host__ __device__ static __forceinline__ __nv_bfloat16 narrow(float x) { return __float2bfloat16_rn(x); }
};
template <>
struct FieldElem<__half> {
  using Compute = float;
  __host__ __device__ static __forceinline__ float widen(__half x) { return __half2float(x); }
  __host__ __device__ static __forceinline__ __half narrow(float x) { return __float2half_rn(x); }
};

template <class T>
struct Tag {
  using type = T;
};
// Calls f(Tag<T>{}) with the C++ type of a field type and returns true; false for any other type.
template <class F>
bool with_field_type(ElemType t, F&& f) {
  switch (t) {
    case ElemType::kFloat: f(Tag<float>{}); return true;
    case ElemType::kDouble: f(Tag<double>{}); return true;
    case ElemType::kBFloat16: f(Tag<__nv_bfloat16>{}); return true;
    case ElemType::kHalf: f(Tag<__half>{}); return true;
    default: return false;
  }
}
// The same, and any other type is an error of `what`.
template <class F>
void with_field_type(ElemType t, const char* what, F&& f) {
  if (!with_field_type(t, f))
    HPCP_FAIL(std::string(what) + ": the field type must be float, double, bfloat16 or half");
}

}  // namespace hpcp
