// Allreduce kernels for the reductions other than the sum: prod, min and max (↔ MPI_PROD / MPI_MIN / MPI_MAX), and on
// the integer types band, bor, bxor, land, lor and lxor (↔ MPI_BAND / MPI_BOR / MPI_BXOR / MPI_LAND / MPI_LOR /
// MPI_LXOR), and on the value-index pair types maxloc and minloc (↔ MPI_MAXLOC / MPI_MINLOC).
//
// They are the kernel templates of ring_allreduce.cuh, the ones the sum runs, instantiated with another combine policy:
// the same loads, stores, arrival / ack words and barriers, in the same combine order.  Two differences on purpose:
//   * the rings OVERWRITE VC (hop 0 stores VA[r] without reading VC), as MPI_Allreduce does; the sum accumulates;
//   * two-shot combines owner first, ((VA[s] o VA[s+1]) o ...), in its tail loop too, so every element has one order.
// Semantics per type (docs/allreduce.md):
//   min / max   integers compare signed or unsigned by type; floats follow IEEE 754-2019 minimum / maximum (any NaN
//               gives NaN, -0 < +0), 16-bit floats in their own format (the result is one of the inputs);
//   prod        integers wrap modulo 2^w (signed and unsigned share the bits, as for the sum); floats round every
//               product to nearest even without FTZ; two-shot multiplies the 16-bit types in fp32 and rounds once;
//   band / bor / bxor   &, |, ^ of the element bits, whatever the width and signedness (one kernel set for all);
//   land / lor / lxor   an element is true iff it is nonzero over its whole width; the result is 0 or 1 of the type.
//   maxloc / minloc     the pair whose value is largest / smallest wins; bit-equal values (or two NaNs) take the smaller
//               signed index.  Values compare signed; floats in max / min's order (-0 < +0, a NaN value wins in both);
//               the padding bytes of a result are zero.
// A NaN result is the type's canonical quiet NaN (all bits set but the sign), the same bits on every rank.
#include "ring_allreduce.cuh"

namespace hpcp {

namespace {

constexpr uint32_t kNaN32 = 0x7fffffffu;
constexpr unsigned long long kNaN64 = 0x7fffffffffffffffull;

__device__ __forceinline__ unsigned long long lane64(uint32_t lo, uint32_t hi) {
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}

// A combine policy from a function of one 32-bit word (L::f) or of one 64-bit lane (L::f64).
template <class L>
struct Words {
  static __device__ __forceinline__ uint4 combine(const uint4& a, const uint4& b) {
    return make_uint4(L::f(a.x, b.x), L::f(a.y, b.y), L::f(a.z, b.z), L::f(a.w, b.w));
  }
};
template <class L>
struct DWords {
  static __device__ __forceinline__ uint4 combine(const uint4& a, const uint4& b) {
    const unsigned long long lo = L::f64(lane64(a.x, a.y), lane64(b.x, b.y));
    const unsigned long long hi = L::f64(lane64(a.z, a.w), lane64(b.z, b.w));
    return make_uint4(static_cast<uint32_t>(lo), static_cast<uint32_t>(lo >> 32), static_cast<uint32_t>(hi),
                      static_cast<uint32_t>(hi >> 32));
  }
};

// Two 16-bit floating lanes: every NaN lane becomes the canonical 0x7fff (kInf = the +inf bits of the format).
template <uint32_t kInf>
__device__ __forceinline__ uint32_t canonical_nan16x2(uint32_t r) {
  const uint32_t nan = __vcmpgtu2(r & 0x7fff7fffu, kInf * 0x10001u);  // 0xffff in every NaN lane
  return (r & ~nan) | (0x7fff7fffu & nan);
}
template <typename H2>
constexpr uint32_t kInf16 = std::is_same<H2, __half2>::value ? 0x7c00u : 0x7f80u;

// ------------------------------------------------------------- min / max ----
// Equal inputs give their bitwise AND (max) or OR (min): the same bits unless they are +0 and -0, and then +0 (max) or
// -0 (min), the order IEEE maximum / minimum demand and the hardware min / max do not promise.
template <bool kMax>
struct MnMxF32 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    float r;  // max.NaN / min.NaN: the canonical NaN if either input is NaN
    if (kMax)
      asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(__uint_as_float(a)), "f"(__uint_as_float(b)));
    else
      asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(__uint_as_float(a)), "f"(__uint_as_float(b)));
    return __uint_as_float(a) == __uint_as_float(b) ? (kMax ? a & b : a | b) : __float_as_uint(r);
  }
};
template <typename H2, bool kMax>
struct MnMxH2 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    const H2 x = *reinterpret_cast<const H2*>(&a), y = *reinterpret_cast<const H2*>(&b);
    const H2 m = kMax ? __hmax2_nan(x, y) : __hmin2_nan(x, y);  // canonical NaN if either lane input is NaN
    const uint32_t eq = __heq2_mask(x, y);
    return (*reinterpret_cast<const uint32_t*>(&m) & ~eq) | ((kMax ? a & b : a | b) & eq);
  }
};
template <bool kMax>
struct MnMxF64 {
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) {
    const double x = __longlong_as_double(static_cast<long long>(a));
    const double y = __longlong_as_double(static_cast<long long>(b));
    if (x != x || y != y) return kNaN64;
    if (x == y) return kMax ? a & b : a | b;
    return (kMax ? x > y : x < y) ? a : b;
  }
};
template <bool kMax>
struct MnMxS32 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    const int x = static_cast<int>(a), y = static_cast<int>(b);
    return static_cast<uint32_t>(kMax ? max(x, y) : min(x, y));
  }
};
template <bool kMax>
struct MnMxU32 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return kMax ? max(a, b) : min(a, b); }
};
template <bool kMax>
struct MnMxS64 {
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) {
    const long long x = static_cast<long long>(a), y = static_cast<long long>(b);
    return (kMax ? x > y : x < y) ? a : b;
  }
};
template <bool kMax>
struct MnMxU64 {
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) {
    return (kMax ? a > b : a < b) ? a : b;
  }
};
template <bool kMax>
struct MnMxS16x2 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return kMax ? __vmaxs2(a, b) : __vmins2(a, b); }
};
template <bool kMax>
struct MnMxU16x2 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return kMax ? __vmaxu2(a, b) : __vminu2(a, b); }
};
template <bool kMax>
struct MnMxU8x4 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return kMax ? __vmaxu4(a, b) : __vminu4(a, b); }
};

// min / max need one class per element type: signed and unsigned integers compare differently.
template <typename T, bool kMax> struct MinMax;
template <bool kMax> struct MinMax<float, kMax> : Words<MnMxF32<kMax>> {};
template <bool kMax> struct MinMax<double, kMax> : DWords<MnMxF64<kMax>> {};
template <bool kMax> struct MinMax<int, kMax> : Words<MnMxS32<kMax>> {};
template <bool kMax> struct MinMax<unsigned int, kMax> : Words<MnMxU32<kMax>> {};
template <bool kMax> struct MinMax<long long, kMax> : DWords<MnMxS64<kMax>> {};
template <bool kMax> struct MinMax<unsigned long long, kMax> : DWords<MnMxU64<kMax>> {};
template <bool kMax> struct MinMax<short, kMax> : Words<MnMxS16x2<kMax>> {};
template <bool kMax> struct MinMax<unsigned short, kMax> : Words<MnMxU16x2<kMax>> {};
template <bool kMax> struct MinMax<unsigned char, kMax> : Words<MnMxU8x4<kMax>> {};
template <bool kMax> struct MinMax<__nv_bfloat16, kMax> : Words<MnMxH2<__nv_bfloat162, kMax>> {};
template <bool kMax> struct MinMax<__half, kMax> : Words<MnMxH2<__half2, kMax>> {};
template <typename T> struct Max : MinMax<T, true> {};
template <typename T> struct Min : MinMax<T, false> {};

// ------------------------------------------------------------------ prod ----
struct MulF32 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    const float r = __fmul_rn(__uint_as_float(a), __uint_as_float(b));
    return r != r ? kNaN32 : __float_as_uint(r);
  }
};
struct MulF64 {
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) {
    const double r = __dmul_rn(__longlong_as_double(static_cast<long long>(a)),
                               __longlong_as_double(static_cast<long long>(b)));
    return r != r ? kNaN64 : static_cast<unsigned long long>(__double_as_longlong(r));
  }
};
template <typename H2>
struct MulH2 {  // one product rounded to nearest even in the 16-bit format per lane, subnormals kept
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    const H2 r = __hmul2_rn(*reinterpret_cast<const H2*>(&a), *reinterpret_cast<const H2*>(&b));
    return canonical_nan16x2<kInf16<H2>>(*reinterpret_cast<const uint32_t*>(&r));
  }
};
struct MulI32 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return a * b; }
};
struct MulI64 {
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) { return a * b; }
};
// The low w bits of a product depend only on the low w bits of its factors.
struct MulI16x2 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    return ((a >> 16) * (b >> 16)) << 16 | ((a * b) & 0xffffu);
  }
};
struct MulU8x4 {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) {
    return ((a >> 24) * (b >> 24)) << 24 | (((a >> 16) * (b >> 16)) & 0xffu) << 16 |
           (((a >> 8) * (b >> 8)) & 0xffu) << 8 | ((a * b) & 0xffu);
  }
};

// prod per addition class (AddClass): signed and unsigned integers share the wrapping product.
template <typename C> struct Prod;
template <> struct Prod<float> : Words<MulF32> {};
template <> struct Prod<double> : DWords<MulF64> {};
template <> struct Prod<int> : Words<MulI32> {};
template <> struct Prod<long long> : DWords<MulI64> {};
template <> struct Prod<short> : Words<MulI16x2> {};
template <> struct Prod<unsigned char> : Words<MulU8x4> {};
template <> struct Prod<__nv_bfloat16> : Words<MulH2<__nv_bfloat162>> {};
template <> struct Prod<__half> : Words<MulH2<__half2>> {};

// Two-shot's 16-bit prod: fp32 products, owner first, rounded once to T, NaN lanes canonical.
struct MulF32Raw {
  static __device__ __forceinline__ float apply(float a, float b) { return __fmul_rn(a, b); }
};
template <typename T>
struct Prod8 : Wide8<T, MulF32Raw> {
  __device__ __forceinline__ uint4 round() const {
    constexpr uint32_t inf = std::is_same<T, __half>::value ? 0x7c00u : 0x7f80u;
    const uint4 r = Wide8<T, MulF32Raw>::round();
    return make_uint4(canonical_nan16x2<inf>(r.x), canonical_nan16x2<inf>(r.y), canonical_nan16x2<inf>(r.z),
                      canonical_nan16x2<inf>(r.w));
  }
};
template <> struct TwoShotInF32<Prod<__nv_bfloat16>> : std::true_type { using acc = Prod8<__nv_bfloat16>; };
template <> struct TwoShotInF32<Prod<__half>> : std::true_type { using acc = Prod8<__half>; };

// ------------------------------------------------- bitwise and logical ----
// Integer types only (dispatch_op refuses the floating ones).  All six are exact, commutative and associative: every
// combine order gives the same bits.

// band / bor / bxor act on the bits alone: one instantiation serves every integer type.
struct AndW {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return a & b; }
};
struct OrW {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return a | b; }
};
struct XorW {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return a ^ b; }
};
struct BAnd : Words<AndW> {};
struct BOr : Words<OrW> {};
struct BXor : Words<XorW> {};

// The lanes of width class C (AddClass): t(x) is 1 in every lane of x that is nonzero over the whole element width (a
// long holding 1 << 40 is true) and 0 in the others.  Two lanes are both true iff their unsigned minimum (umin) is
// nonzero and either is iff their OR is, so land and lor test one value per lane; lxor (x) is lor but not land (for
// bytes on the top bit of each lane before it is normalised).  Each form keeps the push and pull rings within the
// registers of Max of the same width (testing every input on its own costs the narrow lanes two more).
template <typename C> struct Lanes;
template <> struct Lanes<int> {
  static __device__ __forceinline__ uint32_t t(uint32_t x) { return x != 0u; }
  static __device__ __forceinline__ uint32_t umin(uint32_t a, uint32_t b) { return min(a, b); }
  static __device__ __forceinline__ uint32_t x(uint32_t a, uint32_t b) { return t(a | b) ^ t(umin(a, b)); }
};
template <> struct Lanes<long long> {  // the full 64-bit lane, never its 32-bit halves
  using W = unsigned long long;
  static __device__ __forceinline__ W t(W x) { return x != 0ull; }
  static __device__ __forceinline__ W umin(W a, W b) { return min(a, b); }
  static __device__ __forceinline__ W x(W a, W b) { return t(a | b) ^ t(umin(a, b)); }
};
template <> struct Lanes<short> {
  static __device__ __forceinline__ uint32_t t(uint32_t x) { return __vcmpne2(x, 0u) & 0x00010001u; }
  static __device__ __forceinline__ uint32_t umin(uint32_t a, uint32_t b) { return __vminu2(a, b); }
  static __device__ __forceinline__ uint32_t x(uint32_t a, uint32_t b) { return t(a | b) ^ t(umin(a, b)); }
};
template <> struct Lanes<unsigned char> {
  static __device__ __forceinline__ uint32_t t(uint32_t x) { return __vcmpne4(x, 0u) & 0x01010101u; }
  static __device__ __forceinline__ uint32_t umin(uint32_t a, uint32_t b) { return __vminu4(a, b); }
  // (v & 0x7f) + 0x7f carries into the top bit of a byte iff its low bits are nonzero, and | v adds the top bit itself
  static __device__ __forceinline__ uint32_t top(uint32_t v) { return ((v & 0x7f7f7f7fu) + 0x7f7f7f7fu) | v; }
  static __device__ __forceinline__ uint32_t x(uint32_t a, uint32_t b) {
    return ((top(a | b) ^ top(umin(a, b))) >> 7) & 0x01010101u;
  }
};

struct LAndF {
  template <class L, typename W> static __device__ __forceinline__ W g(W a, W b) { return L::t(L::umin(a, b)); }
};
struct LOrF {
  template <class L, typename W> static __device__ __forceinline__ W g(W a, W b) { return L::t(a | b); }
};
struct LXorF {
  template <class L, typename W> static __device__ __forceinline__ W g(W a, W b) { return L::x(a, b); }
};
template <typename C, class F>
struct LogicW {
  static __device__ __forceinline__ uint32_t f(uint32_t a, uint32_t b) { return F::template g<Lanes<C>>(a, b); }
  static __device__ __forceinline__ unsigned long long f64(unsigned long long a, unsigned long long b) {
    return F::template g<Lanes<C>>(a, b);
  }
};
template <typename C, class L> struct LanesOf : Words<L> {};
template <class L> struct LanesOf<long long, L> : DWords<L> {};
template <typename C> struct LAnd : LanesOf<C, LogicW<C, LAndF>> {};
template <typename C> struct LOr : LanesOf<C, LogicW<C, LOrF>> {};
template <typename C> struct LXor : LanesOf<C, LogicW<C, LXorF>> {};

// ------------------------------------------------------- maxloc / minloc ----
// Exact, commutative and associative: a pair's rank is (key of its value, then -index) for maxloc and (key, index) for
// minloc, and the combine returns the better pair, so every combine order selects the same one.  key() is an unsigned
// integer in the order of the values (a NaN value at the top for maxloc, at the bottom for minloc: it wins in both, all
// NaNs tie); canon() is the value's bits as a result stores them (the canonical NaN; a short's upper half zero).
template <typename V> struct LocValue;
template <> struct LocValue<int> {
  using W = uint32_t;
  template <bool kMax> static __device__ __forceinline__ W key(W v) { return v ^ 0x80000000u; }
  static __device__ __forceinline__ W canon(W v) { return v; }
};
template <> struct LocValue<short> {  // the low half of the word, sign-extended for the compare
  using W = uint32_t;
  template <bool kMax> static __device__ __forceinline__ W key(W v) { return (v & 0xffffu) ^ 0x8000u; }
  static __device__ __forceinline__ W canon(W v) { return v & 0xffffu; }
};
template <> struct LocValue<long long> {
  using W = unsigned long long;
  template <bool kMax> static __device__ __forceinline__ W key(W v) { return v ^ 0x8000000000000000ull; }
  static __device__ __forceinline__ W canon(W v) { return v; }
};
// IEEE bits -> a key in their total order (negative values reversed below the positive ones, -0 just below +0).
template <typename W, W kSign, W kInf, W kNaN>
struct LocFloat {
  static __device__ __forceinline__ bool nan(W v) { return (v & ~kSign) > kInf; }
  template <bool kMax> static __device__ __forceinline__ W key(W v) {
    return nan(v) ? (kMax ? ~W{0} : W{0}) : (v & kSign) ? ~v : v | kSign;
  }
  static __device__ __forceinline__ W canon(W v) { return nan(v) ? kNaN : v; }
};
template <> struct LocValue<float> : LocFloat<uint32_t, 0x80000000u, 0x7f800000u, kNaN32> {
  using W = uint32_t;
};
template <> struct LocValue<double>
    : LocFloat<unsigned long long, 0x8000000000000000ull, 0x7ff0000000000000ull, kNaN64> {
  using W = unsigned long long;
};

// a o b on one pair: true if a is the result (the better key, or the same key and the smaller or equal index).
template <typename V, bool kMax>
__device__ __forceinline__ bool loc_takes_a(typename LocValue<V>::W va, uint32_t ia, typename LocValue<V>::W vb,
                                            uint32_t ib) {
  const auto ka = LocValue<V>::template key<kMax>(va), kb = LocValue<V>::template key<kMax>(vb);
  return (kMax ? ka > kb : ka < kb) || (ka == kb && static_cast<int>(ia) <= static_cast<int>(ib));
}
// The 8-byte pairs, two per vector: value in x / z, index in y / w.
template <typename V, bool kMax>
struct Loc8 {
  static __device__ __forceinline__ uint4 combine(const uint4& a, const uint4& b) {
    const bool lo = loc_takes_a<V, kMax>(a.x, a.y, b.x, b.y), hi = loc_takes_a<V, kMax>(a.z, a.w, b.z, b.w);
    return make_uint4(LocValue<V>::canon(lo ? a.x : b.x), lo ? a.y : b.y, LocValue<V>::canon(hi ? a.z : b.z),
                      hi ? a.w : b.w);
  }
};
// The 16-byte pairs, one per vector: value in (x, y), index in z, padding in w.
template <typename V, bool kMax>
struct Loc16 {
  static __device__ __forceinline__ uint4 combine(const uint4& a, const uint4& b) {
    const bool t = loc_takes_a<V, kMax>(lane64(a.x, a.y), a.z, lane64(b.x, b.y), b.z);
    const unsigned long long v = LocValue<V>::canon(t ? lane64(a.x, a.y) : lane64(b.x, b.y));
    return make_uint4(static_cast<uint32_t>(v), static_cast<uint32_t>(v >> 32), t ? a.z : b.z, 0u);
  }
};
template <typename P, bool kMax>
using LocOf = std::conditional_t<sizeof(P) == 16, Loc16<typename P::value_type, kMax>,
                                 Loc8<typename P::value_type, kMax>>;
// P = LocPair<V> (dtype_traits.h).
template <typename P> struct MaxLoc : LocOf<P, true> {};
template <typename P> struct MinLoc : LocOf<P, false> {};

// ---------------------------------------------------------------- kernels ----
// VC = op(VC, VA) over whole vectors; block 0's thread 0 combines the last partial vector in registers and writes back
// only its tail_bytes.
template <class Op>
__global__ void __launch_bounds__(512) combine_kernel(const uint4* __restrict__ va, uint4* __restrict__ vc,
                                                      size_t nvec, const unsigned char* va_tail,
                                                      unsigned char* vc_tail, size_t tail_bytes) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += stride)
    vc[i] = Op::combine(vc[i], ptx::ld_weak_v4(va + i));
  if (blockIdx.x == 0 && threadIdx.x == 0 && tail_bytes > 0) {
    uint4 x = make_uint4(0, 0, 0, 0), acc = x;
    unsigned char* xb = reinterpret_cast<unsigned char*>(&x);
    unsigned char* ab = reinterpret_cast<unsigned char*>(&acc);
    for (size_t k = 0; k < tail_bytes; ++k) xb[k] = va_tail[k], ab[k] = vc_tail[k];
    const uint4 r = Op::combine(acc, x);
    const unsigned char* rb = reinterpret_cast<const unsigned char*>(&r);
    for (size_t k = 0; k < tail_bytes; ++k) vc_tail[k] = rb[k];
  }
}

// The bitwise and logical policies of width class C.
template <typename C, typename F>
void dispatch_bit_op(ReduceOp op, F& f) {
  switch (op) {
    case ReduceOp::kBAnd: f(BAnd{}); break;
    case ReduceOp::kBOr: f(BOr{}); break;
    case ReduceOp::kBXor: f(BXor{}); break;
    case ReduceOp::kLAnd: f(LAnd<C>{}); break;
    case ReduceOp::kLOr: f(LOr<C>{}); break;
    case ReduceOp::kLXor: f(LXor<C>{}); break;
    default: HPCP_FAIL("allreduce ops: not a bitwise or logical op"); break;
  }
}

// Run f(Op{}) with the combine policy of (type, op).  An op that does not reduce the type (the bitwise and logical ops
// on the floating types, maxloc / minloc on any but the pair types, any other op on those) is refused here, before any
// kernel is chosen, as MPI refuses it.
template <typename F>
void dispatch_op(ElemType type, ReduceOp op, F&& f) {
  HPCP_REQUIRE(reduce_op_takes(op, type), reduce_op_type_error(op, type));
  if (elem_type_is_pair(type)) {
    dispatch_pair(type, [&](auto tag) {
      using P = decltype(tag);
      if (op == ReduceOp::kMaxLoc)
        f(MaxLoc<P>{});
      else
        f(MinLoc<P>{});
    });
    return;
  }
  dispatch_elem(type, [&](auto tag) {
    using T = decltype(tag);
    switch (op) {
      case ReduceOp::kMax: f(Max<T>{}); break;
      case ReduceOp::kMin: f(Min<T>{}); break;
      case ReduceOp::kProd: f(Prod<typename AddClass<T>::type>{}); break;
      case ReduceOp::kSum: HPCP_FAIL("allreduce ops: the sum has its own kernels"); break;
      default:
        if constexpr (std::is_integral<T>::value)
          dispatch_bit_op<typename AddClass<T>::type>(op, f);
        else
          HPCP_FAIL(reduce_op_type_error(op, type));
        break;
    }
  });
}

}  // namespace

AllreduceKernels op_allreduce_kernels(ElemType type, ReduceOp op) {
  AllreduceKernels k{};
  dispatch_op(type, op, [&](auto tag) { k = allreduce_kernels_of<decltype(tag), true, true>(); });
  return k;
}

const void* op_combine_kernel(ElemType type, ReduceOp op) {
  const void* k = nullptr;
  dispatch_op(type, op, [&](auto tag) { k = kernel_ptr(combine_kernel<decltype(tag)>); });
  return k;
}

}  // namespace hpcp
