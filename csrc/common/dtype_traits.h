// C++ element type -> runtime descriptor used by the kernels and the bindings.
//
// Plays the role of mpi::get_datatype<T>() in the reference
// (aurora.mpich.miniapps/src/include/mpi_datatype.hpp:18-51: C++ type -> MPI_Datatype,
// default MPI_BYTE).  There is no MPI here; what a collective kernel needs to
// know about T is its size, whether an arithmetic reduction exists for it and a
// printable name.  Every type the reference's trait maps to an MPI_SUM-capable
// datatype (short/int/long/float/double and the unsigned integers, :28-51) has
// SUM kernels here (ring, accumulate, two-shot: csrc/kernels/ring_allreduce.cu);
// `long double` has no device representation on NVIDIA GPUs and, like any other
// type, falls back to "bytes" (copy-only), the analogue of MPI_BYTE.
// The two 16-bit floating types MPICH adds as MPIX_C_BF16 / MPIX_C_FLOAT16
// (__nv_bfloat16, __half) have SUM kernels too: the rings round every add to the
// 16-bit format, two-shot accumulates in fp32 and rounds once (docs/allreduce.md).
// cuda_bf16.h / cuda_fp16.h also compile as plain host C++ (g++), so the host-only
// users of this header need nothing beyond the CUDA include directory.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstddef>
#include <cstdint>
#include <string>
#include <type_traits>

#include "../kernels/api.h"
#include "cuda_check.h"

namespace hpcp {

struct DTypeInfo {
  const char* name;      // "float", "int", ... ; "bytes" for opaque types
  size_t size;           // sizeof(T)
  bool reducible;        // has reduction kernels in this suite: SUM for the arithmetic types, maxloc / minloc only
                         // for the value-index pair types
  ElemType elem;         // valid iff reducible
  const char* torch;     // matching torch dtype name, "" if none
};

template <typename T>
struct dtype_of {
  static constexpr DTypeInfo value{"bytes", sizeof(T), false, ElemType::kFloat, ""};
};

#define HPCP_DTYPE(T, NAME, RED, ELEM, TORCH)                                 \
  template <>                                                                 \
  struct dtype_of<T> {                                                        \
    static constexpr DTypeInfo value{NAME, sizeof(T), RED, ELEM, TORCH};      \
  }

HPCP_DTYPE(float, "float", true, ElemType::kFloat, "float32");
HPCP_DTYPE(int, "int", true, ElemType::kInt, "int32");
HPCP_DTYPE(unsigned int, "unsigned int", true, ElemType::kUInt, "uint32");
HPCP_DTYPE(double, "double", true, ElemType::kDouble, "float64");
HPCP_DTYPE(long, "long", true, ElemType::kLong, "int64");
HPCP_DTYPE(long long, "long", true, ElemType::kLong, "int64");
HPCP_DTYPE(unsigned long, "unsigned long", true, ElemType::kULong, "uint64");
HPCP_DTYPE(unsigned long long, "unsigned long", true, ElemType::kULong, "uint64");
HPCP_DTYPE(short, "short", true, ElemType::kShort, "int16");
HPCP_DTYPE(unsigned short, "unsigned short", true, ElemType::kUShort, "uint16");
HPCP_DTYPE(unsigned char, "unsigned char", true, ElemType::kUChar, "uint8");
HPCP_DTYPE(__nv_bfloat16, "bfloat16", true, ElemType::kBFloat16, "bfloat16");
HPCP_DTYPE(__half, "half", true, ElemType::kHalf, "float16");

// The value-index pairs of MPI_MAXLOC / MPI_MINLOC (↔ MPI_FLOAT_INT, MPI_DOUBLE_INT, MPI_LONG_INT, MPI_2INT,
// MPI_SHORT_INT): the C struct {value; int index;} in its natural layout, the same on the host and the device.  The
// padding (after a short value, after the index of a 16-byte pair) is zero in every pair a combine produces.
template <typename V>
struct LocPair {
  using value_type = V;
  V value;
  int index;
};
static_assert(sizeof(LocPair<float>) == 8 && offsetof(LocPair<float>, index) == 4, "float_int layout");
static_assert(sizeof(LocPair<double>) == 16 && offsetof(LocPair<double>, index) == 8, "double_int layout");
static_assert(sizeof(LocPair<long long>) == 16 && offsetof(LocPair<long long>, index) == 8, "long_int layout");
static_assert(sizeof(LocPair<int>) == 8 && offsetof(LocPair<int>, index) == 4, "2int layout");
static_assert(sizeof(LocPair<short>) == 8 && offsetof(LocPair<short>, index) == 4, "short_int layout");
HPCP_DTYPE(LocPair<float>, "float_int", true, ElemType::kFloatInt, "");
HPCP_DTYPE(LocPair<double>, "double_int", true, ElemType::kDoubleInt, "");
HPCP_DTYPE(LocPair<long long>, "long_int", true, ElemType::kLongInt, "");
HPCP_DTYPE(LocPair<int>, "2int", true, ElemType::kTwoInt, "");
HPCP_DTYPE(LocPair<short>, "short_int", true, ElemType::kShortInt, "");
#undef HPCP_DTYPE

template <typename T>
constexpr DTypeInfo get_dtype(const T& = T{}) {
  return dtype_of<T>::value;
}

// Run-time lookup by name (C++ spelling, torch spelling or a short alias); false if unknown.
inline bool elem_type_from_name(const std::string& name, ElemType* out) {
  struct Row {
    const char* name;
    ElemType type;
  };
  static const Row rows[] = {
      {"float", ElemType::kFloat},    {"float32", ElemType::kFloat},       {"f32", ElemType::kFloat},
      {"int", ElemType::kInt},        {"int32", ElemType::kInt},           {"s32", ElemType::kInt},
      {"uint", ElemType::kUInt},      {"unsigned", ElemType::kUInt},       {"unsigned int", ElemType::kUInt},
      {"uint32", ElemType::kUInt},    {"u32", ElemType::kUInt},
      {"double", ElemType::kDouble},  {"float64", ElemType::kDouble},      {"f64", ElemType::kDouble},
      {"long", ElemType::kLong},      {"int64", ElemType::kLong},          {"s64", ElemType::kLong},
      {"ulong", ElemType::kULong},    {"unsigned long", ElemType::kULong}, {"uint64", ElemType::kULong},
      {"u64", ElemType::kULong},
      {"short", ElemType::kShort},    {"int16", ElemType::kShort},         {"s16", ElemType::kShort},
      {"ushort", ElemType::kUShort},  {"unsigned short", ElemType::kUShort}, {"uint16", ElemType::kUShort},
      {"u16", ElemType::kUShort},
      {"uchar", ElemType::kUChar},    {"unsigned char", ElemType::kUChar}, {"uint8", ElemType::kUChar},
      {"u8", ElemType::kUChar},
      {"bfloat16", ElemType::kBFloat16}, {"bf16", ElemType::kBFloat16},
      {"half", ElemType::kHalf},      {"float16", ElemType::kHalf},        {"f16", ElemType::kHalf},
      {"fp16", ElemType::kHalf},
      {"float_int", ElemType::kFloatInt}, {"double_int", ElemType::kDoubleInt}, {"long_int", ElemType::kLongInt},
      {"2int", ElemType::kTwoInt},    {"int_int", ElemType::kTwoInt},      {"short_int", ElemType::kShortInt},
  };
  for (const Row& r : rows)
    if (name == r.name) {
      *out = r.type;
      return true;
    }
  return false;
}
inline const char* elem_type_name(ElemType t) {
  switch (t) {
    case ElemType::kFloat: return "float";
    case ElemType::kInt: return "int";
    case ElemType::kUInt: return "uint";
    case ElemType::kDouble: return "double";
    case ElemType::kLong: return "long";
    case ElemType::kULong: return "ulong";
    case ElemType::kShort: return "short";
    case ElemType::kUShort: return "ushort";
    case ElemType::kUChar: return "uchar";
    case ElemType::kBFloat16: return "bfloat16";
    case ElemType::kHalf: return "half";
    case ElemType::kFloatInt: return "float_int";
    case ElemType::kDoubleInt: return "double_int";
    case ElemType::kLongInt: return "long_int";
    case ElemType::kTwoInt: return "2int";
    case ElemType::kShortInt: return "short_int";
  }
  return "?";
}

inline bool elem_type_is_pair(ElemType t) {
  return t == ElemType::kFloatInt || t == ElemType::kDoubleInt || t == ElemType::kLongInt || t == ElemType::kTwoInt ||
         t == ElemType::kShortInt;
}

// Run f(T{}) with the C++ type of `t`, one of the eleven arithmetic types; a pair type is refused (dispatch_pair).
template <typename F>
void dispatch_elem(ElemType t, F&& f) {
  switch (t) {
    case ElemType::kFloat: f(float{}); break;
    case ElemType::kInt: f(int{}); break;
    case ElemType::kUInt: f(static_cast<unsigned int>(0)); break;
    case ElemType::kDouble: f(double{}); break;
    case ElemType::kLong: f(static_cast<long long>(0)); break;
    case ElemType::kULong: f(static_cast<unsigned long long>(0)); break;
    case ElemType::kShort: f(static_cast<short>(0)); break;
    case ElemType::kUShort: f(static_cast<unsigned short>(0)); break;
    case ElemType::kUChar: f(static_cast<unsigned char>(0)); break;
    case ElemType::kBFloat16: f(__nv_bfloat16{}); break;
    case ElemType::kHalf: f(__half{}); break;
    case ElemType::kFloatInt:
    case ElemType::kDoubleInt:
    case ElemType::kLongInt:
    case ElemType::kTwoInt:
    case ElemType::kShortInt:
      HPCP_FAIL(std::string(elem_type_name(t)) + " is a value-index pair type: only maxloc and minloc reduce it");
  }
}

// Run f(LocPair<V>{}) with the pair struct of `t`; an arithmetic type is refused.
template <typename F>
void dispatch_pair(ElemType t, F&& f) {
  switch (t) {
    case ElemType::kFloatInt: f(LocPair<float>{}); break;
    case ElemType::kDoubleInt: f(LocPair<double>{}); break;
    case ElemType::kLongInt: f(LocPair<long long>{}); break;
    case ElemType::kTwoInt: f(LocPair<int>{}); break;
    case ElemType::kShortInt: f(LocPair<short>{}); break;
    default: HPCP_FAIL(std::string(elem_type_name(t)) + " is not a value-index pair type");
  }
}

// C++ element type -> the addition class its sum kernels are instantiated for: signed and unsigned integers of one
// width share the add (and the wrapping product).
template <typename T> struct AddClass { using type = T; };
template <> struct AddClass<unsigned int> { using type = int; };
template <> struct AddClass<unsigned long long> { using type = long long; };
template <> struct AddClass<unsigned short> { using type = short; };

// Run f(C{}) with the addition class of `t` (eight kernel instantiations instead of eleven).
template <typename F>
void dispatch_add_class(ElemType t, F&& f) {
  dispatch_elem(t, [&](auto tag) { f(typename AddClass<decltype(tag)>::type{}); });
}

// The 16-bit floating types: two-shot accumulates them in fp32 and rounds once.
template <typename T>
constexpr bool kSum16InF32 = std::is_same<T, __nv_bfloat16>::value || std::is_same<T, __half>::value;

// Reduction by name: sum, prod (or product), min, max, band, bor, bxor, land, lor, lxor, maxloc, minloc; false if
// unknown.
inline bool reduce_op_from_name(const std::string& name, ReduceOp* out) {
  if (name == "sum") *out = ReduceOp::kSum;
  else if (name == "prod" || name == "product") *out = ReduceOp::kProd;
  else if (name == "min") *out = ReduceOp::kMin;
  else if (name == "max") *out = ReduceOp::kMax;
  else if (name == "band") *out = ReduceOp::kBAnd;
  else if (name == "bor") *out = ReduceOp::kBOr;
  else if (name == "bxor") *out = ReduceOp::kBXor;
  else if (name == "land") *out = ReduceOp::kLAnd;
  else if (name == "lor") *out = ReduceOp::kLOr;
  else if (name == "lxor") *out = ReduceOp::kLXor;
  else if (name == "maxloc") *out = ReduceOp::kMaxLoc;
  else if (name == "minloc") *out = ReduceOp::kMinLoc;
  else return false;
  return true;
}
inline const char* reduce_op_name(ReduceOp op) {
  switch (op) {
    case ReduceOp::kSum: return "sum";
    case ReduceOp::kProd: return "prod";
    case ReduceOp::kMin: return "min";
    case ReduceOp::kMax: return "max";
    case ReduceOp::kBAnd: return "band";
    case ReduceOp::kBOr: return "bor";
    case ReduceOp::kBXor: return "bxor";
    case ReduceOp::kLAnd: return "land";
    case ReduceOp::kLOr: return "lor";
    case ReduceOp::kLXor: return "lxor";
    case ReduceOp::kMaxLoc: return "maxloc";
    case ReduceOp::kMinLoc: return "minloc";
  }
  return "?";
}

// The bitwise and logical ops reduce the integer types only, as in MPI.
inline bool reduce_op_integer_only(ReduceOp op) {
  return op == ReduceOp::kBAnd || op == ReduceOp::kBOr || op == ReduceOp::kBXor || op == ReduceOp::kLAnd ||
         op == ReduceOp::kLOr || op == ReduceOp::kLXor;
}
inline bool elem_type_is_integer(ElemType t) {
  return t != ElemType::kFloat && t != ElemType::kDouble && t != ElemType::kBFloat16 && t != ElemType::kHalf &&
         !elem_type_is_pair(t);
}
// maxloc and minloc reduce the pair types only, and they are the only ops that do.
inline bool reduce_op_on_pairs(ReduceOp op) { return op == ReduceOp::kMaxLoc || op == ReduceOp::kMinLoc; }
// Whether `op` reduces `t`.
inline bool reduce_op_takes(ReduceOp op, ElemType t) {
  if (elem_type_is_pair(t) || reduce_op_on_pairs(op)) return elem_type_is_pair(t) && reduce_op_on_pairs(op);
  return !reduce_op_integer_only(op) || elem_type_is_integer(t);
}
// The refusal of an op that does not reduce a type (reduce_op_takes), the same words in every layer.
inline std::string reduce_op_type_error(ReduceOp op, ElemType t) {
  if (elem_type_is_pair(t))
    return std::string("op must be maxloc or minloc for ") + elem_type_name(t) + ": " + reduce_op_name(op) +
           " reduces arithmetic types only";
  if (reduce_op_on_pairs(op))
    return std::string("op must be ") +
           (elem_type_is_integer(t) ? "sum, prod, min, max, band, bor, bxor, land, lor or lxor" : "sum, prod, min or max") +
           " for " + elem_type_name(t) + ": " + reduce_op_name(op) + " reduces value-index pair types only";
  return std::string("op must be sum, prod, min or max for ") + elem_type_name(t) + ": " + reduce_op_name(op) +
         " reduces integer types only";
}

}  // namespace hpcp
