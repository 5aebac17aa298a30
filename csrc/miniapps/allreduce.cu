// allreduce — the miniapp: ring "rotate + accumulate" allreduce of a replicated
// array, or a one-launch collective with -a.
//
// Capability parity with the three reference variants
//   mpi-sycl/allreduce-mpi-sycl.cpp:88-215
//   mpi-omp-offload/allreduce-usm-mpi-omp-offload.cpp:78-225
//   mpi-omp-offload/allreduce-map-mpi-omp-offload.cpp:67-179
// Options kept: -h, -a (use the collective), -p k (2^k elements, default 25),
// -H / -D / -S allocation kind (pinned host / device / managed), element type
// float or int (upstream: compile-time APP_DATA_TYPE -> here --type or the
// binary-name suffix `allreduce.float` / `allreduce.int`, like the upstream
// target names `<app>.<type>`).  Output kept: `Passed <rank>` per rank, exit 0.
// bfloat16 / half (`allreduce.bfloat16`, `allreduce.half`, ↔ MPIX_C_BF16 / MPIX_C_FLOAT16): the rings round every add to
// the 16-bit format, -a runs two-shot with fp32 accumulation; the constant-data check stays exact up to P = 16.
// Additions: the elapsed time the reference computes but never prints
// (allreduce-mpi-sycl.cpp:185-190) is printed as max over ranks, with bus GB/s.
//
// Algorithms (--algo):
//   ring          fused K-ring: all P-1 exchanges + P accumulations in one launch/rank
//   ring-unfused  same data movement as the reference with separate kernels:
//                 rendezvous put kernel, then Accumulate kernel, per step (VA/VB swap)
//   ring-rsag     bandwidth-optimal ring: reduce-scatter + all-gather in one launch/rank,
//                 2(P-1)/P of the block sent per rank (n padded to whole 16-byte vectors x P)
//   (with -a)     nvls when NVSwitch multicast is available, else two-shot P2P;
//                 force with --coll nvls|twoshot
// Reductions (--op, ↔ MPI_SUM / MPI_PROD / MPI_MIN / MPI_MAX): sum (default) accumulates into VC; prod, min and max
// overwrite VC and run on every algorithm except nvls (sum-only; -a picks two-shot for them).  Each op has its own
// constant-data check, exact in every type up to P = 16: max (rank r holds r) -> P-1, min (P-r) -> 1, prod (2 on the
// odd ranks below 8, else 1) -> 2^min(P/2, 4).
// On the integer types only (↔ MPI_BAND ... MPI_LXOR; a floating --type is a usage error): band, bor, bxor, land, lor
// and lxor, same rules.  Their checks (docs/allreduce.md) are exact in uchar and tell the bitwise from the logical op at
// every P >= 2: band (255 - 2^(r mod 4)) -> 256 - 2^min(P,4), bor (2^(r mod 4)) -> 2^min(P,4) - 1, bxor (128 on rank 0,
// r elsewhere) -> 128 ^ 1 ^ ... ^ (P-1), land (r+1) -> 1, lor (2(r mod 2)) -> 1, lxor (3 on rank 0, else 0) -> 1; at
// P = 1 VC is VA.
// On the value-index pair types only (--type float_int|double_int|long_int|2int|short_int or allreduce.<pair type>, ↔
// MPI_MAXLOC / MPI_MINLOC on MPI_FLOAT_INT ...): maxloc (the default op there) and minloc, same rules; any other op on a
// pair type, and maxloc / minloc on any other type, is a usage error.  Their check is exact bytes, padding included:
// maxloc (rank 0 holds (0, -P-10), rank r (1, 2r-3), VC starts at (7, -1000)) -> (1, -1), minloc with the values 1 and 0
// (VC (-7, -1000)) -> (0, -1); at P = 1 VC is VA.  A tie broken towards the larger index, an unsigned index compare, a
// selection by index alone and a kernel that reads VC each give another pair.
//
// Run as `reduce_scatter` (a program-name link to this binary) it is the stand-alone reduce-scatter (↔
// MPI_Reduce_scatter_block, ncclReduceScatter; launch_reduce_scatter): every rank's send buffer holds P segments of n
// elements (-p k: 2^k elements padded to P whole 16-byte segments, as -a pads) and rank r receives op over p of segment r
// of rank p's, owner first.  Options: --type, --op, -p, -n, --iters, --warmup, --ctas, --json, --cpu; device memory
// only, so -a, --algo, --coll, --slots, --pull, -H, -S, -R (and --chunk, --map-alias, --profile-relaunch) are usage
// errors.  Check: the allreduce's constant data, except that for the sum segment q of rank p holds p + (q mod 8), so
// rank r expects P(P-1)/2 + P*(r mod 8) (exact in every type up to P = 16) and a rank that reduced a neighbour's segment
// fails; the receive buffer starts as a value no rank expects (251 for the sum, whose vc_init 0 is rank 0's result at
// P = 1), and the send buffer is checked unchanged.  --cpu runs the same owner-first fold on host threads.
#include <cuda_profiler_api.h>
#include <getopt.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
#include <string>
#include <vector>

#include "../common/cuda_check.h"
#include "../common/dtype_traits.h"
#include "../common/nvtx.h"
#include "../common/peer_mem.h"
#include "../common/rank_runtime.h"
#include "../common/signal_layout.h"
#include "../kernels/api.h"
#include "../kernels/ring_order.h"
#include "devices.hpp"

namespace {

using namespace hpcp;


struct Config {
  int ranks = 0;
  int log2_elems = 25;
  bool use_collective = false;
  AllocKind kind = AllocKind::kDevice;
  ElemType type = ElemType::kFloat;
  ReduceOp op = ReduceOp::kSum;
  bool op_given = false;  // no --op: sum, or maxloc on a pair type
  std::string algo = "ring";
  std::string coll = "auto";
  int iters = 5;
  bool profile_relaunch = false;  // rank 0 repeats its last launch between cudaProfilerStart/Stop
  int warmup = 1;
  int ctas = 0;
  size_t chunk_elems = 0;
  uint64_t timeout_ns = 30ull * 1000 * 1000 * 1000;
  std::string json_path;
  int slots = 0;     // --slots 2: the reference's VA/VB double buffer with per-chunk acks (default: P-1 slots)
  bool pull = false; // --pull: the fused ring moves its bytes as peer LOADS (receiver-driven) instead of peer stores
  bool cpu = false;  // --cpu: host-only plumbing run (threads as ranks, memcpy as send/recv)
  // -R: the reference's `map` variant (allreduce-map-mpi-omp-offload.cpp:113-115,159,168-170): the arrays are host
  // malloc'ed; `target enter data map(alloc)` gives each a DEVICE-RESIDENT copy the kernels and the exchange work on
  // (use_device_ptr, :38); `target update from(VC)` brings the result back and the HOST verifies it.  Here: malloc +
  // cudaMalloc pair, explicit cudaMemcpy D2H as the update.  --map-alias keeps round 1's zero-copy variant instead
  // (cudaHostRegister + device alias: every access crosses PCIe).
  bool map_alias = false;
};

void print_help() {
  std::cout << "Usage: allreduce [options]\n"
               "options:\n"
               " -p k        2^k elements per rank            default: 25\n"
               " -a          one-launch collective (NVLS multimem / two-shot P2P) instead of the ring\n"
               " -H          pinned host memory   (cudaHostAlloc)\n"
               " -D          device memory        (cudaMalloc, default)\n"
               " -S          managed memory       (cudaMallocManaged)\n"
               " -R          the `map` variant of the reference: host malloc'ed arrays with a device-resident mapped copy\n"
               "             (kernels and the exchange use the device copy; VC is updated back and verified on the host)\n"
               " --map-alias with -R: map by cudaHostRegister + device alias instead (zero-copy over PCIe)\n"
               " --profile-relaunch    after the run rank 0 repeats its last launch (same epochs, peers idle) between\n"
               "                       cudaProfilerStart/Stop: use with `ncu --profile-from-start off`\n"
               " -n N        ranks (one host thread + one GPU each; default: all GPUs;\n"
               "             more ranks than GPUs are placed round-robin)\n"
               " --type T   element type: float int uint double long ulong short ushort uchar bfloat16 half,\n"
               "            or a value-index pair: float_int double_int long_int 2int short_int\n"
               "            (default float, or binary-name suffix)\n"
               " --algo ring|ring-unfused|ring-rsag   fused persistent ring kernel (default),\n"
               "                            separate put + accumulate kernels per step, or the\n"
               "                            bandwidth-optimal reduce-scatter + all-gather ring\n"
               " --coll auto|nvls|twoshot   collective used with -a\n"
               " --op sum|prod|min|max      reduction (default sum; nvls is sum-only, -a uses two-shot for the others)\n"
               "    |band|bor|bxor|land|lor|lxor   bitwise and logical reductions: integer types only\n"
               "    |maxloc|minloc   value-index reductions: pair types only (their default op is maxloc)\n"
               " --iters N --warmup N  timed / untimed repetitions (min is reported)\n"
               " --ctas N --chunk N    kernel tuning (CTAs per rank, elements per ring chunk)\n"
               " --pull                fused ring, receiver-driven: every block is LOADED from the left neighbour's\n"
               "                       memory (loads issued by the receiver instead of the sender's stores)\n"
               " --slots 2             fused ring with two receive slots + per-chunk acks (the reference's VA/VB\n"
               "                       double buffer) instead of P-1 slots without flow control\n"
               " --json FILE           append one JSON row\n"
               " --cpu                 host-only plumbing run: ranks are threads, send/recv are memcpy\n";
}

struct Shared {
  Config cfg;
  NodeMemory* mem = nullptr;
  size_t n = 0;
  size_t n_chunks = 0;
  size_t pad_extra = 0;  // words after the fixed pad: arrival words (+ ack words with --slots 2)
  uint32_t epoch_advance = 0;  // arrival epochs one launch of the fused ring uses
  SymmetricBuffer va, vb, vc, slots, pads;
  MulticastBuffer mc_va, mc_vc;
  std::vector<void*> host_va, host_vc;  // -R: the host arrays whose mapped copies are va / vc
  bool nvls = false;
  double best_ms = 0;
  unsigned long long total_bad = 0;
};

// Host arithmetic of the 16-bit floating types: exact widening to fp32, and an add that is one fp32 add rounded once to
// nearest even in the 16-bit format (fp32 has more than 2p+2 bits, so that equals the correctly rounded 16-bit add the
// ring kernels do).  Every other type keeps its own arithmetic.
template <typename T>
double host_to_double(T x) {
  return static_cast<double>(x);
}
double host_to_double(__nv_bfloat16 x) { return __bfloat162float(x); }
double host_to_double(__half x) { return __half2float(x); }
template <typename T>
T host_add(T a, T b) {
  return static_cast<T>(a + b);
}
__nv_bfloat16 host_add(__nv_bfloat16 a, __nv_bfloat16 b) {
  return __float2bfloat16_rn(__bfloat162float(a) + __bfloat162float(b));
}
__half host_add(__half a, __half b) { return __float2half_rn(__half2float(a) + __half2float(b)); }
template <typename T>
T host_from_float(float x) {
  return static_cast<T>(x);
}
template <>
__nv_bfloat16 host_from_float(float x) { return __float2bfloat16_rn(x); }
template <>
__half host_from_float(float x) { return __float2half_rn(x); }

// The kernels' NaN result: all bits set but the sign (little-endian: the sign bit is in the last byte).
template <typename T>
T host_canonical_nan() {
  T x;
  std::memset(static_cast<void*>(&x), 0xff, sizeof x);
  reinterpret_cast<unsigned char*>(&x)[sizeof x - 1] = 0x7f;
  return x;
}

// op(a, b) with the kernels' semantics (docs/allreduce.md): integers compare by their own signedness and multiply
// modulo 2^w; floats follow IEEE maximum / minimum (NaN wins, -0 < +0) and round every product once; the 16-bit floats
// compare exactly and round every product to their format (from its exact fp64 value); NaN results are canonical.
// The bitwise ops act on the bits; the logical ones take an element as true iff it is nonzero and give 0 or 1.
template <typename T>
T host_combine(ReduceOp op, T a, T b) {
  if (op == ReduceOp::kSum) return host_add(a, b);
  if constexpr (std::is_integral<T>::value) {
    switch (op) {
      case ReduceOp::kProd:
        return static_cast<T>(static_cast<unsigned long long>(a) * static_cast<unsigned long long>(b));
      case ReduceOp::kBAnd: return static_cast<T>(a & b);
      case ReduceOp::kBOr: return static_cast<T>(a | b);
      case ReduceOp::kBXor: return static_cast<T>(a ^ b);
      case ReduceOp::kLAnd: return static_cast<T>(a != 0 && b != 0);
      case ReduceOp::kLOr: return static_cast<T>(a != 0 || b != 0);
      case ReduceOp::kLXor: return static_cast<T>((a != 0) != (b != 0));
      default: break;
    }
    return op == ReduceOp::kMax ? std::max(a, b) : std::min(a, b);
  } else {
    const double x = host_to_double(a), y = host_to_double(b);
    if (std::isnan(x) || std::isnan(y)) return host_canonical_nan<T>();
    if (op == ReduceOp::kProd) {
      T r;
      if constexpr (std::is_same<T, __nv_bfloat16>::value)
        r = __double2bfloat16(x * y);
      else if constexpr (std::is_same<T, __half>::value)
        r = __double2half(x * y);
      else
        r = a * b;
      return std::isnan(host_to_double(r)) ? host_canonical_nan<T>() : r;
    }
    if (x == y) return (std::signbit(x) == (op == ReduceOp::kMax)) ? b : a;  // +-0: max takes +0, min -0
    return (op == ReduceOp::kMax) == (x > y) ? a : b;
  }
}

// Constant-data check of every op: what rank r holds and what every element of the result must equal (exact up to
// P = 16 in every type).
// The integer-only ops' values fit in uchar, and each bitwise op's result differs from its logical twin's at P >= 2.
double op_input(ReduceOp op, int r, int P) {
  switch (op) {
    case ReduceOp::kSum: return r;
    case ReduceOp::kMax: return r;
    case ReduceOp::kMin: return P - r;
    case ReduceOp::kProd: return r % 2 == 1 && r < 8 ? 2 : 1;
    case ReduceOp::kBAnd: return 255 - (1 << (r % 4));
    case ReduceOp::kBOr: return 1 << (r % 4);
    case ReduceOp::kBXor: return r == 0 ? 128 : r;
    case ReduceOp::kLAnd: return r + 1;
    case ReduceOp::kLOr: return 2 * (r % 2);
    case ReduceOp::kLXor: return r == 0 ? 3 : 0;
    case ReduceOp::kMaxLoc:
    case ReduceOp::kMinLoc: break;  // pairs: loc_input
  }
  return 0;
}
double op_expected(ReduceOp op, int P) {
  int x = 128;
  switch (op) {
    case ReduceOp::kSum: return 0.5 * P * (P - 1);
    case ReduceOp::kMax: return P - 1;
    case ReduceOp::kMin: return 1;
    case ReduceOp::kProd: return std::ldexp(1.0, std::min(P / 2, 4));
    case ReduceOp::kBAnd: return 256 - (1 << std::min(P, 4));
    case ReduceOp::kBOr: return (1 << std::min(P, 4)) - 1;
    case ReduceOp::kBXor:
      for (int r = 1; r < P; ++r) x ^= r;
      return x;
    case ReduceOp::kLAnd: return 1;
    case ReduceOp::kLOr: return P >= 2 ? 1 : 0;
    case ReduceOp::kLXor: return P >= 2 ? 1 : 3;  // one rank: VC is VA, unnormalised
    case ReduceOp::kMaxLoc:
    case ReduceOp::kMinLoc: break;  // pairs: loc_expected
  }
  return 0;
}
// VC before the run: 0 for the sum, which accumulates into it; for the other ops a value that would change the result
// if a kernel read VC instead of overwriting it.
double op_vc_init(ReduceOp op, int P) {
  switch (op) {
    case ReduceOp::kMax: return P;
    case ReduceOp::kBOr: return 16;
    case ReduceOp::kBXor: return 64;
    case ReduceOp::kLOr: return 3;
    case ReduceOp::kLXor: return 5;
    default: return 0;
  }
}
// The constant-data check of maxloc / minloc: (value, index) of rank r, of the result and of VC before the run.
struct LocDatum {
  double value;
  int index;
};
LocDatum loc_input(ReduceOp op, int r, int P) {
  const bool mx = op == ReduceOp::kMaxLoc;
  return r == 0 ? LocDatum{mx ? 0.0 : 1.0, -P - 10} : LocDatum{mx ? 1.0 : 0.0, 2 * r - 3};
}
LocDatum loc_expected(ReduceOp op, int P) {
  return P == 1 ? loc_input(op, 0, 1) : LocDatum{op == ReduceOp::kMaxLoc ? 1.0 : 0.0, -1};
}
LocDatum loc_vc_init(ReduceOp op) { return {op == ReduceOp::kMaxLoc ? 7.0 : -7.0, -1000}; }

// The pair with padding bytes zero.
template <typename V>
LocPair<V> host_pair(double value, int index) {
  LocPair<V> p;
  std::memset(static_cast<void*>(&p), 0, sizeof p);
  p.value = static_cast<V>(value);
  p.index = index;
  return p;
}
// maxloc / minloc with the kernels' rules: the larger (maxloc) or smaller (minloc) value wins, a NaN value wins in both,
// -0 < +0; bit-equal values or two NaNs take the smaller signed index; the result has zero padding and a canonical NaN.
template <typename V>
LocPair<V> host_combine(ReduceOp op, LocPair<V> a, LocPair<V> b) {
  const bool mx = op == ReduceOp::kMaxLoc;
  int better = 0;  // > 0: a's value wins, < 0: b's, 0: a tie
  if constexpr (std::is_floating_point<V>::value) {
    const bool na = std::isnan(a.value), nb = std::isnan(b.value);
    if (na || nb)
      better = na == nb ? 0 : na ? 1 : -1;
    else if (a.value != b.value || std::signbit(a.value) != std::signbit(b.value))
      better = ((a.value > b.value || (a.value == b.value && std::signbit(b.value))) == mx) ? 1 : -1;
  } else {
    if (a.value != b.value) better = ((a.value > b.value) == mx) ? 1 : -1;
  }
  const LocPair<V>& w = better > 0 || (better == 0 && a.index <= b.index) ? a : b;
  LocPair<V> r = host_pair<V>(0, w.index);
  if constexpr (std::is_floating_point<V>::value)
    r.value = std::isnan(w.value) ? host_canonical_nan<V>() : w.value;
  else
    r.value = w.value;
  return r;
}
template <typename V>
LocPair<V> host_add(LocPair<V>, LocPair<V>) {
  HPCP_FAIL("the value-index pair types have no sum");
}

// The constant-data inputs and check in the host twin's element type.
template <typename T>
T host_input(ReduceOp op, int r, int P) {
  return static_cast<T>(op_input(op, r, P));
}
template <typename T>
T host_vc_init(ReduceOp op, int P) {
  return static_cast<T>(op_vc_init(op, P));
}
template <typename T>
bool host_is_expected(const T& v, ReduceOp op, int P) {
  return std::abs(host_to_double(v) - host_to_double(static_cast<T>(op_expected(op, P)))) < 1e-6;
}
// The constant data of the host twin for a pair type (the arithmetic types: ArithHost).
template <typename V>
struct PairHost {
  static LocPair<V> input(ReduceOp op, int r, int P) {
    const LocDatum d = loc_input(op, r, P);
    return host_pair<V>(d.value, d.index);
  }
  static LocPair<V> vc_init(ReduceOp op, int) {
    const LocDatum d = loc_vc_init(op);
    return host_pair<V>(d.value, d.index);
  }
  // The value's bits and the index: a struct copy need not keep padding bytes, so the host twin cannot check them.
  static bool is_expected(const LocPair<V>& v, ReduceOp op, int P) {
    const LocDatum d = loc_expected(op, P);
    const V want = static_cast<V>(d.value);
    return std::memcmp(&v.value, &want, sizeof want) == 0 && v.index == d.index;
  }
};
// The bytes of the pair (value, index) with zero padding, written in place.
template <typename V>
void pair_bytes(double value, int index, unsigned char* out) {
  std::memset(out, 0, sizeof(LocPair<V>));
  const V v = static_cast<V>(value);
  std::memcpy(out + offsetof(LocPair<V>, value), &v, sizeof v);
  std::memcpy(out + offsetof(LocPair<V>, index), &index, sizeof index);
}

// The JSON rows carry "op" only when it is not the sum (sum rows keep their shape).
std::string op_json(ReduceOp op) {
  return op == ReduceOp::kSum ? std::string() : std::string(",\"op\":\"") + reduce_op_name(op) + "\"";
}

// A pair type: its value.
double first_element_as_double(const void* p, ElemType t) {
  double x = 0;
  if (elem_type_is_pair(t))
    dispatch_pair(t, [&](auto tag) { x = static_cast<double>(static_cast<const decltype(tag)*>(p)->value); });
  else
    dispatch_elem(t, [&](auto tag) { x = host_to_double(*static_cast<const decltype(tag)*>(p)); });
  return x;
}

template <typename T>
unsigned long long count_mismatch_typed(const void* p, size_t n, double expected) {
  const T* v = static_cast<const T*>(p);
  unsigned long long bad = 0;
  for (size_t i = 0; i < n; ++i) {
    const double d = host_to_double(v[i]) - expected;
    bad += !(d < 1e-6 && d > -1e-6);
  }
  return bad;
}
unsigned long long count_mismatch_on_host(const void* p, size_t n, double expected, ElemType t) {
  unsigned long long bad = n;
  dispatch_elem(t, [&](auto tag) { bad = count_mismatch_typed<decltype(tag)>(p, n, expected); });
  return bad;
}
// Pair types: elements whose bytes differ from the constant-data result of `op`, padding included.
unsigned long long count_pair_mismatch_on_host(const void* p, size_t n, ReduceOp op, int P, ElemType t) {
  unsigned long long bad = n;
  dispatch_pair(t, [&](auto tag) {
    using V = typename decltype(tag)::value_type;
    const LocDatum d = loc_expected(op, P);
    unsigned char want[sizeof(LocPair<V>)];
    pair_bytes<V>(d.value, d.index, want);
    const unsigned char* v = static_cast<const unsigned char*>(p);
    bad = 0;
    for (size_t i = 0; i < n; ++i) bad += std::memcmp(v + i * sizeof want, want, sizeof want) != 0;
  });
  return bad;
}

uint32_t* pad_of(const Shared& sh, int r) { return static_cast<uint32_t*>(sh.pads.ptr[r]); }

void rank_main(RankCtx& ctx, Shared& sh) {
  const Config& cfg = sh.cfg;
  const int me = ctx.rank, P = ctx.world;
  const int dev = sh.mem->device(me);
  HPCP_CUDA(cudaSetDevice(dev));
  cudaStream_t stream;
  HPCP_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  const int right = (me + 1) % P, left = (me - 1 + P) % P;
  const size_t esz = elem_size(cfg.type);
  const bool pair = elem_type_is_pair(cfg.type);
  uint32_t* my_pad = pad_of(sh, me);
  uint32_t* status = my_pad + kPadWords + sh.pad_extra;
  std::vector<uint32_t*> pad_list;
  for (int r = 0; r < P; ++r) pad_list.push_back(pad_of(sh, r));

  void* va = sh.nvls ? sh.mc_va.uc[me] : sh.va.ptr[me];
  void* vc = sh.nvls ? sh.mc_vc.uc[me] : sh.vc.ptr[me];

  uint32_t barrier_epoch = 0, ticket_issued = 0, ring_epoch = 0, step_epoch = 0;
  cudaEvent_t e0, e1;
  HPCP_CUDA(cudaEventCreate(&e0));
  HPCP_CUDA(cudaEventCreate(&e1));
  double best_ms = std::numeric_limits<double>::max();

  // One allreduce on `stream`.  replay = enqueue the PREVIOUS launch again with the same epochs: every word it would
  // wait for is already there, so it moves the same bytes over the same links without needing a running peer —
  // the shape a kernel-replay profiler can capture (--profile-relaunch).
  auto launch_once = [&](bool replay) {
    if (cfg.use_collective) {
      if (!replay) ++barrier_epoch;
      if (sh.nvls) {
        NvlsArgs a;
        a.va_mc = sh.mc_va.mc;
        a.vc_mc = sh.mc_vc.mc;
        for (int r = 0; r < P; ++r) a.pads[r] = pad_list[r];
        a.ticket = my_pad + kPadLocal;
        a.ticket_base = ticket_issued;
        a.rank = me;
        a.world = P;
        a.n = sh.n;
        a.barrier_epoch = barrier_epoch;
        a.timeout_ns = cfg.timeout_ns;
        a.status = status;
        a.op = cfg.op;
        ticket_issued += launch_allreduce_nvls(a, cfg.type, cfg.ctas, dev, stream);
      } else {
        TwoShotArgs a;
        for (int r = 0; r < P; ++r) {
          a.va[r] = sh.va.ptr[r];
          a.vc[r] = sh.vc.ptr[r];
          a.pads[r] = pad_list[r];
        }
        a.ticket = my_pad + kPadLocal;
        a.ticket_base = ticket_issued;
        a.rank = me;
        a.world = P;
        a.n = sh.n;
        a.barrier_epoch = barrier_epoch;
        a.timeout_ns = cfg.timeout_ns;
        a.status = status;
        a.op = cfg.op;
        ticket_issued += launch_allreduce_two_shot(a, cfg.type, cfg.ctas, dev, stream);
      }
    } else if (cfg.algo == "ring") {
      RingArgs a;
      a.va = va;
      a.vc = vc;
      a.slots_local = sh.slots.ptr[me];
      a.slots_right = sh.slots.ptr[right];
      a.arrived_local = my_pad + kPadWords;
      a.arrived_right = pad_of(sh, right) + kPadWords;
      a.world = P;
      a.n = sh.n;
      a.chunk_elems = cfg.chunk_elems;
      a.epoch_base = replay ? ring_epoch - sh.epoch_advance : ring_epoch;
      a.timeout_ns = cfg.timeout_ns;
      a.status = status;
      a.n_slots = cfg.slots;
      a.op = cfg.op;
      if (cfg.pull) {  // receiver-driven: load from the left neighbour instead of being stored into
        a.pull = true;
        a.va_left = sh.va.ptr[left];
        a.slots_left = sh.slots.ptr[left];
      }
      if (cfg.slots == 2) {  // ack words follow the arrival words on every pad
        a.ack_local = my_pad + kPadWords + sh.n_chunks;
        a.ack_left = pad_of(sh, left) + kPadWords + sh.n_chunks;
      }
      if (!replay) ring_epoch += sh.epoch_advance;
      launch_ring_allreduce(a, cfg.type, cfg.ctas, dev, stream);
    } else if (cfg.algo == "ring-rsag") {
      RingRsAgArgs a;
      a.va = va;
      a.vc = vc;
      a.slots_local = sh.slots.ptr[me];
      a.slots_right = sh.slots.ptr[right];
      a.vc_right = sh.vc.ptr[right];
      a.arrived_local = my_pad + kPadWords;
      a.arrived_right = pad_of(sh, right) + kPadWords;
      a.rank = me;
      a.world = P;
      a.n = sh.n;
      a.chunk_elems = cfg.chunk_elems;
      a.epoch_base = replay ? ring_epoch - sh.epoch_advance : ring_epoch;
      a.timeout_ns = cfg.timeout_ns;
      a.status = status;
      a.phases = kRsAgAllreduce;
      a.op = cfg.op;
      if (!replay) ring_epoch += sh.epoch_advance;
      launch_ring_rsag(a, cfg.type, cfg.ctas, dev, stream);
    } else {  // ring-unfused: the reference's step structure with separate kernels
      HPCP_REQUIRE(!replay, "--profile-relaunch supports the one-launch algorithms only");
      void* cur = va;
      void* other = sh.vb.ptr[me];
      void* right_cur = sh.va.ptr[right];     // what the right neighbour currently calls VA
      void* right_other = sh.vb.ptr[right];   // ... and VB (where my block must land)
      if (cfg.op == ReduceOp::kSum)
        launch_accumulate(cur, vc, sh.n, cfg.type, stream);
      else  // the other ops overwrite VC: step 0 is VC = VA
        HPCP_CUDA(cudaMemcpyAsync(vc, cur, sh.n * esz, cudaMemcpyDeviceToDevice, stream));
      for (int s = 1; s < P; ++s) {
        ++step_epoch;
        // Post the receive: my VB is free (my previous put from it has completed in-stream).
        launch_signal(pad_of(sh, left) + kPadReady + me, step_epoch, stream);
        SyncOps sync;
        sync.wait_flag = my_pad + kPadReady + right;
        sync.wait_epoch = step_epoch;
        sync.signal_flag = pad_of(sh, right) + kPadDone + me;
        sync.signal_epoch = step_epoch;
        sync.ticket = my_pad + kPadLocal;
        sync.ticket_base = ticket_issued;
        sync.timeout_ns = cfg.timeout_ns;
        sync.status = status;
        CopyTuning tune;
        tune.ctas = cfg.ctas;
        ticket_issued += launch_copy(right_other, cur, sh.n * esz, false, CopyEngine::kLdSt, tune, sync,
                                     dev, stream);
        launch_wait(my_pad + kPadDone + left, step_epoch, cfg.timeout_ns, status, stream);
        std::swap(cur, other);
        std::swap(right_cur, right_other);
        launch_accumulate(cur, vc, sh.n, cfg.type, stream, cfg.op);
      }
    }

  };

  for (int it = 0; it < cfg.warmup + cfg.iters; ++it) {
    NvtxRange iter_range(it < cfg.warmup ? "allreduce warm-up" : "allreduce timed");
    // (Re-)initialise outside the timed region: VA = VB = rank (the op's input), VC = 0 (sum) or a poison value.
    void* vb = cfg.algo == "ring-unfused" && !cfg.use_collective ? sh.vb.ptr[me] : nullptr;
    if (pair) {
      const LocDatum x = loc_input(cfg.op, me, P), c = loc_vc_init(cfg.op);
      launch_init_pair(va, sh.n, x.value, x.index, cfg.type, stream);
      if (vb) launch_init_pair(vb, sh.n, x.value, x.index, cfg.type, stream);
      launch_init_pair(vc, sh.n, c.value, c.index, cfg.type, stream);
    } else {
      const double x = op_input(cfg.op, me, P);
      launch_init3(va, vb, vc, sh.n, x, x, op_vc_init(cfg.op, P), cfg.type, stream);
    }
    HPCP_CUDA(cudaStreamSynchronize(stream));
    ctx.barrier();
    launch_barrier_all(pad_list.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
    HPCP_CUDA(cudaEventRecord(e0, stream));

    launch_once(false);

    HPCP_CUDA(cudaEventRecord(e1, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    uint32_t st = 0;
    HPCP_CUDA(cudaMemcpy(&st, status, sizeof st, cudaMemcpyDeviceToHost));
    HPCP_REQUIRE(st == 0, "rank " + std::to_string(me) + ": device-side wait timed out");
    float ms = 0;
    HPCP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double t = ctx.max(ms);
    if (it >= cfg.warmup) best_ms = std::min(best_ms, t);
  }

  // Verify: every element of VC equals P(P-1)/2 (sum), or the op's constant result.
  const double want = op_expected(cfg.op, P);
  unsigned long long bad = 0;
  const bool mapped_copy = !sh.host_vc.empty();
  if (mapped_copy) {
    // `#pragma omp target update from(VC[:n])` (allreduce-map-mpi-omp-offload.cpp:159), then the host checks its
    // own array (:163-164) and prints "<rank> <VC[0]>" (:161).
    HPCP_CUDA(cudaMemcpyAsync(sh.host_vc[me], vc, sh.n * esz, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    bad = pair ? count_pair_mismatch_on_host(sh.host_vc[me], sh.n, cfg.op, P, cfg.type)
               : count_mismatch_on_host(sh.host_vc[me], sh.n, want, cfg.type);
  } else {
    unsigned long long* count = nullptr;
    HPCP_CUDA(cudaMalloc(&count, sizeof *count));
    HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
    if (pair) {
      const LocDatum w = loc_expected(cfg.op, P);
      launch_count_pair_mismatch(vc, sh.n, w.value, w.index, cfg.type, count, stream);
    } else {
      launch_count_mismatch(vc, sh.n, want, cfg.type, count, stream);
    }
    HPCP_CUDA(cudaMemcpyAsync(&bad, count, sizeof bad, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    (void)cudaFree(count);
  }
  const double total_bad = ctx.sum(static_cast<double>(bad));
  if (bad == 0)
    std::cout << "Passed " << me << std::endl;
  else
    std::cout << "FAILED " << me << ": " << bad << " wrong elements" << std::endl;
  if (mapped_copy)
    std::cout << me << " " << first_element_as_double(sh.host_vc[me], cfg.type) << std::endl;
  else if (cfg.kind == AllocKind::kMapped && !sh.nvls)  // --map-alias: the buffer IS host memory, read in place
    std::cout << me << " " << first_element_as_double(vc, cfg.type) << std::endl;
  if (cfg.profile_relaunch) {
    // Profilers that replay one kernel many times serialise the process's kernels, and a replayed pass would wait for
    // peers that are long done.  Rank 0 therefore re-enqueues its last launch with the SAME epochs between
    // cudaProfilerStart/Stop while every other rank is idle: `ncu --profile-from-start off` captures exactly that one.
    ctx.barrier();
    if (me == 0) {
      HPCP_CUDA(cudaProfilerStart());
      launch_once(true);
      HPCP_CUDA(cudaStreamSynchronize(stream));
      HPCP_CUDA(cudaProfilerStop());
      uint32_t st = 0;
      HPCP_CUDA(cudaMemcpy(&st, status, sizeof st, cudaMemcpyDeviceToHost));
      HPCP_REQUIRE(st == 0, "profile relaunch: device-side wait timed out");
      std::cout << "# profile relaunch of rank 0 done (same epochs, peers idle)" << std::endl;
    }
    ctx.barrier();
  }
  if (me == 0) {
    sh.best_ms = best_ms;
    sh.total_bad = static_cast<unsigned long long>(total_bad);
  }
  (void)cudaEventDestroy(e0);
  (void)cudaEventDestroy(e1);
  (void)cudaStreamDestroy(stream);
}


// ---------------------------------------------------------------- host-only path ----
// The reference pattern on the CPU: ranks are threads of the rank runtime, "send to the right
// neighbour" is a memcpy into its VB, the collective is a direct sum over every rank's VA.  No GPU,
// no kernels: this is the plumbing configuration used to test the program logic (options, ring
// order, verification, output) on a machine without a device.
// --algo ring-rsag runs the hops of ring_rsag_kernel with the same rules (ring_order.h): whole segments are memcpy'd
// into the right neighbour's slot or VC, with a barrier between hops.
// H supplies the constant data: input(op, r, P), vc_init(op, P) and is_expected(v, op, P).
template <typename T>
struct ArithHost {
  static T input(ReduceOp op, int r, int P) { return host_input<T>(op, r, P); }
  static T vc_init(ReduceOp op, int P) { return host_vc_init<T>(op, P); }
  static bool is_expected(const T& v, ReduceOp op, int P) { return host_is_expected(v, op, P); }
};

template <typename T, class H>
int run_on_host_typed(const Config& cfg) {
  const int P = cfg.ranks > 0 ? cfg.ranks : 4;
  const bool rsag = cfg.algo == "ring-rsag" && !cfg.use_collective;
  size_t n = size_t{1} << cfg.log2_elems;
  const size_t unit = 16 / sizeof(T) * static_cast<size_t>(P);
  if (rsag && n % unit != 0) n = (n / unit + 1) * unit;  // whole 16-byte vectors per segment, as on the device
  const size_t seg_n = n / P;
  std::vector<std::vector<T>> va(P), vb(P), vc(P);
  double elapsed_ms = 0;
  unsigned long long total_bad = 0;
  const ReduceOp op = cfg.op;
  run_ranks(P, [&](RankCtx& ctx) {
    const int me = ctx.rank, right = (me + 1) % P;
    va[me].assign(n, H::input(op, me, P));
    vb[me].assign(n, H::input(op, me, P));
    vc[me].assign(n, H::vc_init(op, P));
    ctx.barrier();
    const auto t0 = std::chrono::steady_clock::now();
    if (cfg.use_collective && op != ReduceOp::kSum) {
      // two-shot's op rule: element i belongs to slice s = i*P/n, whose owner combines VA[s], VA[s+1], ... (ranks mod
      // P) in that order; the 16-bit prod multiplies in fp32 and rounds once
      for (size_t i = 0; i < n; ++i) {
        const int s = static_cast<int>(i * P / n);
        if constexpr (kSum16InF32<T>) {
          if (op == ReduceOp::kProd) {
            float acc = static_cast<float>(host_to_double(va[s][i]));
            for (int q = 1; q < P; ++q) acc *= static_cast<float>(host_to_double(va[(s + q) % P][i]));
            vc[me][i] = std::isnan(acc) ? host_canonical_nan<T>() : host_from_float<T>(acc);
            continue;
          }
        }
        T acc = va[s][i];
        for (int q = 1; q < P; ++q) acc = host_combine(op, acc, va[(s + q) % P][i]);
        vc[me][i] = acc;
      }
    } else if (cfg.use_collective && kSum16InF32<T>) {
      // two-shot's 16-bit rule: element i belongs to slice s = i*P/n, whose owner s sums VA[s], VA[s+1], ... (ranks
      // mod P) in fp32 and rounds once
      if constexpr (kSum16InF32<T>) {
        for (size_t i = 0; i < n; ++i) {
          const int s = static_cast<int>(i * P / n);
          float acc = static_cast<float>(host_to_double(va[s][i]));
          for (int q = 1; q < P; ++q) acc += static_cast<float>(host_to_double(va[(s + q) % P][i]));
          vc[me][i] = static_cast<T>(acc);
        }
      }
    } else if (cfg.use_collective) {
      for (int r = 0; r < P; ++r)
        for (size_t i = 0; i < n; ++i) vc[me][i] = host_add(vc[me][i], va[r][i]);
    } else if (rsag) {
      vb[me].resize(seg_n * std::max(P - 1, 1));  // receive slots
      ctx.barrier();
      std::vector<T> x(seg_n);
      for (int h = 0; h <= rsag_last_hop(kRsAgAllreduce, P); ++h) {
        const size_t seg = static_cast<size_t>(rsag_segment(h, me, P)) * seg_n;
        const T* src = (rsag_reads_vc(h, P) ? vc[me].data() : va[me].data()) + seg;
        const int rs = rsag_src_slot(h, kRsAgAllreduce, P);
        for (size_t i = 0; i < seg_n; ++i)
          x[i] = rs >= 0 ? host_combine(op, vb[me][rs * seg_n + i], src[i]) : src[i];
        if (rsag_writes_own_vc(h, P)) std::memcpy(vc[me].data() + seg, x.data(), seg_n * sizeof(T));
        if (rsag_forwards(h, kRsAgAllreduce, P)) {
          const int fs = rsag_fwd_slot(h, P);
          T* dst = fs >= 0 ? vb[right].data() + fs * seg_n : vc[right].data() + seg;
          std::memcpy(dst, x.data(), seg_n * sizeof(T));  // "send right"
        }
        ctx.barrier();  // the hop has landed everywhere
      }
    } else {
      if (op == ReduceOp::kSum)
        for (size_t i = 0; i < n; ++i) vc[me][i] = host_add(vc[me][i], va[me][i]);
      else  // the other ops overwrite VC
        vc[me] = va[me];
      for (int s = 1; s < P; ++s) {
        std::memcpy(vb[right].data(), va[me].data(), n * sizeof(T));  // "send right"
        ctx.barrier();                                                 // everybody received
        va[me].swap(vb[me]);
        ctx.barrier();                                                 // nobody still reads the old VA
        for (size_t i = 0; i < n; ++i) vc[me][i] = host_combine(op, vc[me][i], va[me][i]);
      }
    }
    const double ms =
        std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const double t = ctx.max(ms);
    unsigned long long bad = 0;
    for (size_t i = 0; i < n; ++i) bad += !H::is_expected(vc[me][i], op, P);
    const double all_bad = ctx.sum(static_cast<double>(bad));
    if (bad == 0)
      std::cout << "Passed " << me << std::endl;
    else
      std::cout << "FAILED " << me << ": " << bad << " wrong elements" << std::endl;
    if (me == 0) {
      elapsed_ms = t;
      total_bad = static_cast<unsigned long long>(all_bad);
    }
  });
  std::cout << "Elapsed (max over ranks): " << elapsed_ms << " ms | "
            << (cfg.use_collective ? "collective" : rsag ? "host-ring-rsag" : "ring") << " " << elem_type_name(cfg.type)
            << " host-threads P=" << P << " N=2^" << cfg.log2_elems << " arrays=" << alloc_kind_name(cfg.kind)
            << (op != ReduceOp::kSum ? std::string(" op=") + reduce_op_name(op) : std::string())
            << " (host vectors in this mode)" << std::endl;
  if (!cfg.json_path.empty()) {  // same row shape as the GPU path; the algo name marks the plumbing run
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      const double sent = cfg.use_collective ? 0.0
                          : rsag             ? 2.0 * (P - 1) / P * n * sizeof(T)
                                             : static_cast<double>(P - 1) * n * sizeof(T);
      std::fprintf(f,
                   "{\"pattern\":\"allreduce\",\"algo\":\"%s\",\"type\":\"%s\",\"alloc\":\"host-vectors\","
                   "\"ranks\":%d,\"elements\":%zu,\"ms\":%.6f,\"GBps_sent_per_rank\":%.3f,\"mismatches\":%llu%s}\n",
                   cfg.use_collective ? "host-collective" : rsag ? "host-ring-rsag" : "host-ring",
                   elem_type_name(cfg.type), P, n, elapsed_ms,
                   elapsed_ms > 0 ? sent / (elapsed_ms * 1e6) : 0.0, total_bad, op_json(op).c_str());
      std::fclose(f);
    }
  }
  return total_bad == 0 ? 0 : 1;
}

int run_on_host(const Config& cfg) {
  int rc = 1;
  if (elem_type_is_pair(cfg.type))
    dispatch_pair(cfg.type, [&](auto tag) {
      using T = decltype(tag);
      rc = run_on_host_typed<T, PairHost<typename T::value_type>>(cfg);
    });
  else
    dispatch_elem(cfg.type, [&](auto tag) { rc = run_on_host_typed<decltype(tag), ArithHost<decltype(tag)>>(cfg); });
  return rc;
}

// ---------------------------------------------------------------------------------------------- reduce-scatter ----
constexpr double kRsSumPoison = 251;  // above every rank's sum up to P = 16 (at most 232), exact in every type

double rs_input(ReduceOp op, int p, int q, int P) { return op == ReduceOp::kSum ? p + q % 8 : op_input(op, p, P); }
double rs_expected(ReduceOp op, int r, int P) {
  return op == ReduceOp::kSum ? 0.5 * P * (P - 1) + P * (r % 8) : op_expected(op, P);
}
double rs_poison(ReduceOp op, int P) { return op == ReduceOp::kSum ? kRsSumPoison : op_vc_init(op, P); }

// Elements per segment: 2^log2 padded to P whole 16-byte segments, divided by P.
size_t rs_segment(const Config& cfg, int P) {
  const size_t unit = 16 / elem_size(cfg.type) * static_cast<size_t>(P);
  const size_t total = ((size_t{1} << cfg.log2_elems) + unit - 1) / unit * unit;
  return total / P;
}

void rs_report(const Config& cfg, int P, size_t n, double ms, unsigned long long bad, bool host) {
  const double sent = static_cast<double>(P - 1) * n * elem_size(cfg.type);
  const double gbps = ms > 0 ? sent / (ms * 1e-3) * 1e-9 : 0.0;
  const char* algo = host ? "host" : "direct";
  std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << ms << " ms | reduce_scatter " << algo << " "
            << elem_type_name(cfg.type) << " P=" << P << " n=" << n << " op=" << reduce_op_name(cfg.op)
            << (host ? " host-threads" : "") << " | " << gbps << " GB/s sent per rank" << std::endl;
  if (!cfg.json_path.empty()) {
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      std::fprintf(f,
                   "{\"pattern\":\"reduce_scatter\",\"algo\":\"%s\",\"type\":\"%s\",\"op\":\"%s\",\"ranks\":%d,"
                   "\"elements\":%zu,\"ms\":%.6f,\"GBps_sent_per_rank\":%.3f,\"mismatches\":%llu}\n",
                   algo, elem_type_name(cfg.type), reduce_op_name(cfg.op), P, n, ms, gbps, bad);
      std::fclose(f);
    }
  }
}

void rs_print_verdict(int me, unsigned long long bad) {
  const std::string line = bad == 0 ? "Passed " + std::to_string(me) + "\n"
                                    : "FAILED " + std::to_string(me) + ": " + std::to_string(bad) + " wrong elements\n";
  std::cout << line << std::flush;
}

struct RsShared {
  Config cfg;
  NodeMemory* mem = nullptr;
  size_t n = 0;
  SymmetricBuffer send, recv, pads;
  double best_ms = 0;
  unsigned long long total_bad = 0;
};

// Fill n elements at p with the constant datum of (op, rank p's value x) / (pair) on the stream.
void rs_fill(void* p, size_t n, ReduceOp op, int rank, int P, double x, const Config& cfg, cudaStream_t st) {
  if (elem_type_is_pair(cfg.type)) {
    const LocDatum d = loc_input(op, rank, P);
    launch_init_pair(p, n, d.value, d.index, cfg.type, st);
  } else {
    launch_init3(p, nullptr, nullptr, n, x, 0, 0, cfg.type, st);
  }
}

void rs_rank_main(RankCtx& ctx, RsShared& sh) {
  const Config& cfg = sh.cfg;
  const int me = ctx.rank, P = ctx.world;
  const int dev = sh.mem->device(me);
  HPCP_CUDA(cudaSetDevice(dev));
  cudaStream_t stream;
  HPCP_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  std::vector<uint32_t*> pads;
  for (int r = 0; r < P; ++r) pads.push_back(static_cast<uint32_t*>(sh.pads.ptr[r]));
  uint32_t* status = pads[me] + kPadWords;
  const size_t n = sh.n, seg = n * elem_size(cfg.type);
  unsigned char* my_send = static_cast<unsigned char*>(sh.send.ptr[me]);
  void* my_recv = sh.recv.ptr[me];
  const bool pair = elem_type_is_pair(cfg.type);
  unsigned long long* count = nullptr;
  HPCP_CUDA(cudaMalloc(&count, sizeof *count));
  cudaEvent_t e0, e1;
  HPCP_CUDA(cudaEventCreate(&e0));
  HPCP_CUDA(cudaEventCreate(&e1));
  uint32_t barrier_epoch = 0, ticket_issued = 0;
  double best = std::numeric_limits<double>::max();
  for (int it = 0; it < cfg.warmup + cfg.iters; ++it) {
    NvtxRange range(it < cfg.warmup ? "reduce_scatter warm-up" : "reduce_scatter timed");
    for (int q = 0; q < P; ++q) rs_fill(my_send + q * seg, n, cfg.op, me, P, rs_input(cfg.op, me, q, P), cfg, stream);
    if (pair) {
      const LocDatum c = loc_vc_init(cfg.op);
      launch_init_pair(my_recv, n, c.value, c.index, cfg.type, stream);
    } else {
      launch_init3(my_recv, nullptr, nullptr, n, rs_poison(cfg.op, P), 0, 0, cfg.type, stream);
    }
    HPCP_CUDA(cudaStreamSynchronize(stream));
    ctx.barrier();
    launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
    HPCP_CUDA(cudaEventRecord(e0, stream));
    ReduceScatterArgs a;
    for (int r = 0; r < P; ++r) {
      a.send[r] = sh.send.ptr[r];
      a.pads[r] = pads[r];
    }
    a.recv = my_recv;
    a.ticket = pads[me] + kPadLocal;
    a.ticket_base = ticket_issued;
    a.rank = me;
    a.world = P;
    a.n = n;
    a.barrier_epoch = ++barrier_epoch;
    a.timeout_ns = cfg.timeout_ns;
    a.status = status;
    a.op = cfg.op;
    ticket_issued += static_cast<uint32_t>(launch_reduce_scatter(a, cfg.type, cfg.ctas, dev, stream));
    HPCP_CUDA(cudaEventRecord(e1, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    uint32_t st = 0;
    HPCP_CUDA(cudaMemcpy(&st, status, sizeof st, cudaMemcpyDeviceToHost));
    HPCP_REQUIRE(st == 0, "rank " + std::to_string(me) + ": device-side wait timed out");
    float ms = 0;
    HPCP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double t = ctx.max(ms);
    if (it >= cfg.warmup) best = std::min(best, t);
  }
  // The result, and every send segment unchanged.
  HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
  if (pair) {
    const LocDatum w = loc_expected(cfg.op, P), x = loc_input(cfg.op, me, P);
    launch_count_pair_mismatch(my_recv, n, w.value, w.index, cfg.type, count, stream);
    for (int q = 0; q < P; ++q) launch_count_pair_mismatch(my_send + q * seg, n, x.value, x.index, cfg.type, count, stream);
  } else {
    launch_count_mismatch(my_recv, n, rs_expected(cfg.op, me, P), cfg.type, count, stream);
    for (int q = 0; q < P; ++q)
      launch_count_mismatch(my_send + q * seg, n, rs_input(cfg.op, me, q, P), cfg.type, count, stream);
  }
  unsigned long long bad = 0;
  HPCP_CUDA(cudaMemcpyAsync(&bad, count, sizeof bad, cudaMemcpyDeviceToHost, stream));
  HPCP_CUDA(cudaStreamSynchronize(stream));
  const double all_bad = ctx.sum(static_cast<double>(bad));
  rs_print_verdict(me, bad);
  if (me == 0) {
    sh.best_ms = best;
    sh.total_bad = static_cast<unsigned long long>(all_bad);
  }
  (void)cudaFree(count);
  (void)cudaEventDestroy(e0);
  (void)cudaEventDestroy(e1);
  (void)cudaStreamDestroy(stream);
}

// The host twin: rank r folds segment r of every rank owner first, ((S_r[r] o S_{r+1}[r]) o ...), the 16-bit sum and
// prod in fp32 rounded once, as the kernel does; H supplies the pair or arithmetic constant data.
template <typename T>
T rs_host_datum(ReduceOp op, int p, int q, int P) {
  if constexpr (std::is_class<T>::value && !std::is_same<T, __nv_bfloat16>::value && !std::is_same<T, __half>::value) {
    const LocDatum d = loc_input(op, p, P);
    return host_pair<typename T::value_type>(d.value, d.index);
  } else {
    return static_cast<T>(rs_input(op, p, q, P));
  }
}
template <typename T>
bool rs_host_expected(const T& v, ReduceOp op, int r, int P) {
  if constexpr (std::is_class<T>::value && !std::is_same<T, __nv_bfloat16>::value && !std::is_same<T, __half>::value) {
    return PairHost<typename T::value_type>::is_expected(v, op, P);
  } else {
    return std::abs(host_to_double(v) - host_to_double(static_cast<T>(rs_expected(op, r, P)))) < 1e-6;
  }
}

template <typename T>
int rs_run_on_host_typed(const Config& cfg) {
  const int P = cfg.ranks > 0 ? cfg.ranks : 4;
  const size_t n = rs_segment(cfg, P);
  const ReduceOp op = cfg.op;
  std::vector<std::vector<T>> send(P), recv(P);
  double best = std::numeric_limits<double>::max();
  unsigned long long total_bad = 0;
  run_ranks(P, [&](RankCtx& ctx) {
    const int me = ctx.rank;
    send[me].resize(P * n);
    recv[me].resize(n);
    for (int it = 0; it < cfg.warmup + cfg.iters; ++it) {
      for (int q = 0; q < P; ++q) std::fill(send[me].begin() + q * n, send[me].begin() + (q + 1) * n, rs_host_datum<T>(op, me, q, P));
      if constexpr (std::is_class<T>::value && !std::is_same<T, __nv_bfloat16>::value && !std::is_same<T, __half>::value)
        std::fill(recv[me].begin(), recv[me].end(), PairHost<typename T::value_type>::vc_init(op, P));
      else
        std::fill(recv[me].begin(), recv[me].end(), static_cast<T>(rs_poison(op, P)));
      ctx.barrier();
      const auto t0 = std::chrono::steady_clock::now();
      const T* own = send[me].data() + me * n;
      for (size_t i = 0; i < n; ++i) {
        if constexpr (kSum16InF32<T>) {
          if (op == ReduceOp::kSum || op == ReduceOp::kProd) {
            float acc = static_cast<float>(host_to_double(own[i]));
            for (int k = 1; k < P; ++k) {
              const float x = static_cast<float>(host_to_double(send[(me + k) % P][me * n + i]));
              acc = op == ReduceOp::kSum ? acc + x : acc * x;
            }
            recv[me][i] = std::isnan(acc) ? host_canonical_nan<T>() : host_from_float<T>(acc);
            continue;
          }
        }
        T acc = own[i];
        for (int k = 1; k < P; ++k) acc = host_combine(op, acc, send[(me + k) % P][me * n + i]);
        recv[me][i] = acc;
      }
      ctx.barrier();  // the node barrier: every rank has finished reading my send buffer
      const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      const double t = ctx.max(ms);
      if (it >= cfg.warmup) best = std::min(best, t);
    }
    unsigned long long bad = 0;
    for (size_t i = 0; i < n; ++i) bad += !rs_host_expected(recv[me][i], op, me, P);
    for (int q = 0; q < P; ++q)
      for (size_t i = 0; i < n; ++i) {
        const T want = rs_host_datum<T>(op, me, q, P);
        if constexpr (std::is_class<T>::value && !std::is_same<T, __nv_bfloat16>::value && !std::is_same<T, __half>::value)
          bad += std::memcmp(&send[me][q * n + i].value, &want.value, sizeof want.value) != 0 ||
                 send[me][q * n + i].index != want.index;  // a struct copy need not keep the padding bytes
        else
          bad += std::memcmp(&send[me][q * n + i], &want, sizeof want) != 0;
      }
    const double all_bad = ctx.sum(static_cast<double>(bad));
    rs_print_verdict(me, bad);
    if (me == 0) total_bad = static_cast<unsigned long long>(all_bad);
  });
  rs_report(cfg, P, n, best, total_bad, true);
  return total_bad == 0 ? 0 : 1;
}

int run_reduce_scatter(Config cfg) {
  if (elem_type_is_pair(cfg.type) && !cfg.op_given) cfg.op = ReduceOp::kMaxLoc;
  HPCP_REQUIRE(reduce_op_takes(cfg.op, cfg.type), reduce_op_type_error(cfg.op, cfg.type));
  if (cfg.cpu) {
    const int P = cfg.ranks > 0 ? cfg.ranks : 4;
    if (const char* why = reduce_scatter_refusal(P, rs_segment(cfg, P), cfg.type)) HPCP_FAIL(why);
    int rc = 1;
    if (elem_type_is_pair(cfg.type))
      dispatch_pair(cfg.type, [&](auto tag) { rc = rs_run_on_host_typed<decltype(tag)>(cfg); });
    else
      dispatch_elem(cfg.type, [&](auto tag) { rc = rs_run_on_host_typed<decltype(tag)>(cfg); });
    return rc;
  }
  if (cfg.ranks > 0)
    if (const char* why = reduce_scatter_refusal(cfg.ranks, rs_segment(cfg, cfg.ranks), cfg.type)) HPCP_FAIL(why);
  const int ndev = visible_device_count();
  if (ndev == 0) {
    std::cerr << "Error: No devices" << std::endl;
    return 1;
  }
  if (cfg.ranks <= 0) cfg.ranks = std::min(ndev, kApiMaxRanks);
  const int P = cfg.ranks;
  std::vector<int> devices;
  for (int r = 0; r < P; ++r) devices.push_back(primary_device(r, P, ndev));
  const int ranks_per_dev = (P + ndev - 1) / ndev;
  if (ranks_per_dev > 1 && cfg.ctas == 0)  // every rank's barrier CTA must find a slot next to its peers' grids
    cfg.ctas = std::max(1, device_sm_count(devices[0]) / ranks_per_dev);
  NodeMemory mem(devices);
  RsShared sh;
  sh.cfg = cfg;
  sh.mem = &mem;
  sh.n = rs_segment(cfg, P);
  const size_t seg = sh.n * elem_size(cfg.type);
  sh.pads = mem.alloc_pads(0);
  sh.send = mem.alloc(seg * P, AllocKind::kDevice, /*zero=*/false);
  sh.recv = mem.alloc(seg, AllocKind::kDevice, /*zero=*/false);
  run_ranks(P, [&](RankCtx& ctx) { rs_rank_main(ctx, sh); });
  mem.free(sh.send);
  mem.free(sh.recv);
  mem.free(sh.pads);
  rs_report(cfg, P, sh.n, sh.best_ms, sh.total_bad, false);
  return sh.total_bad == 0 ? 0 : 1;
}
}  // namespace

int main(int argc, char** argv) {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  try {
    Shared sh;
    Config& cfg = sh.cfg;
    bool reduce_scatter = false;
    std::string rs_refused;  // the first option the reduce-scatter personality refuses
    // Type from the binary name suffix (`allreduce.int`), like upstream's `<app>.<type>` targets.
    {
      const std::string self = argv[0];
      const auto dot = self.rfind('.');
      if (dot != std::string::npos) (void)elem_type_from_name(self.substr(dot + 1), &cfg.type);
      // Program-name personalities of the reference's three miniapps: their default allocation kinds.
      //   allreduce-mpi-sycl.<type>             shared USM           (allreduce-mpi-sycl.cpp:104)      -> -S
      //   allreduce-usm-mpi-omp-offload.<type>  omp_target_alloc     (allreduce-usm-mpi-omp-offload.cpp:93) -> -D
      //   allreduce-map-mpi-omp-offload.<type>  host arrays + map clause                               -> -R
      const std::string base = self.substr(self.find_last_of('/') + 1);
      if (base.rfind("allreduce-mpi-sycl", 0) == 0) cfg.kind = AllocKind::kManaged;
      if (base.rfind("allreduce-usm-", 0) == 0) cfg.kind = AllocKind::kDevice;
      if (base.rfind("allreduce-map-", 0) == 0) cfg.kind = AllocKind::kMapped;
      reduce_scatter = base == "reduce_scatter";
    }
    static const option long_opts[] = {{"type", required_argument, nullptr, 1},
                                       {"algo", required_argument, nullptr, 2},
                                       {"coll", required_argument, nullptr, 3},
                                       {"iters", required_argument, nullptr, 4},
                                       {"warmup", required_argument, nullptr, 5},
                                       {"ctas", required_argument, nullptr, 6},
                                       {"chunk", required_argument, nullptr, 7},
                                       {"json", required_argument, nullptr, 8},
                                       {"cpu", no_argument, nullptr, 9},
                                       {"slots", required_argument, nullptr, 10},
                                       {"pull", no_argument, nullptr, 11},
                                       {"map-alias", no_argument, nullptr, 12},
                                       {"profile-relaunch", no_argument, nullptr, 13},
                                       {"op", required_argument, nullptr, 14},
                                       {"help", no_argument, nullptr, 'h'},
                                       {nullptr, 0, nullptr, 0}};
    int opt;
    while ((opt = getopt_long(argc, argv, "haHDSRp:n:", long_opts, nullptr)) != -1) {
      if (rs_refused.empty()) {
        switch (opt) {
          case 'a': rs_refused = "-a"; break;
          case 'H': rs_refused = "-H"; break;
          case 'S': rs_refused = "-S"; break;
          case 'R': rs_refused = "-R"; break;
          case 2: rs_refused = "--algo"; break;
          case 3: rs_refused = "--coll"; break;
          case 7: rs_refused = "--chunk"; break;
          case 10: rs_refused = "--slots"; break;
          case 11: rs_refused = "--pull"; break;
          case 12: rs_refused = "--map-alias"; break;
          case 13: rs_refused = "--profile-relaunch"; break;
          default: break;
        }
      }
      switch (opt) {
        case 'h': print_help(); return 1;
        case 'a': cfg.use_collective = true; break;
        case 'H': cfg.kind = AllocKind::kPinned; break;
        case 'D': cfg.kind = AllocKind::kDevice; break;
        case 'S': cfg.kind = AllocKind::kManaged; break;
        case 'R': cfg.kind = AllocKind::kMapped; break;
        case 'p': cfg.log2_elems = std::atoi(optarg); break;
        case 'n': cfg.ranks = std::atoi(optarg); break;
        case 1:
          if (!elem_type_from_name(optarg, &cfg.type)) HPCP_FAIL(std::string("unsupported --type ") + optarg);
          break;
        case 2: cfg.algo = optarg; break;
        case 3: cfg.coll = optarg; break;
        case 4: cfg.iters = std::max(1, std::atoi(optarg)); break;
        case 5: cfg.warmup = std::max(0, std::atoi(optarg)); break;
        case 6: cfg.ctas = std::atoi(optarg); break;
        case 7: cfg.chunk_elems = static_cast<size_t>(std::atoll(optarg)); break;
        case 8: cfg.json_path = optarg; break;
        case 9: cfg.cpu = true; break;
        case 12: cfg.map_alias = true; break;
        case 13: cfg.profile_relaunch = true; break;
        case 14:
          if (!reduce_op_from_name(optarg, &cfg.op))
            HPCP_FAIL(std::string("unknown --op ") + optarg +
                      " (sum|prod|min|max|band|bor|bxor|land|lor|lxor|maxloc|minloc)");
          cfg.op_given = true;
          break;
        case 10: cfg.slots = std::atoi(optarg); break;
        case 11: cfg.pull = true; break;
        default: print_help(); return 1;
      }
    }
    if (reduce_scatter) {
      HPCP_REQUIRE(rs_refused.empty(), "reduce_scatter: " + rs_refused +
                                           " is an allreduce option (the reduce-scatter runs one kernel on device memory)");
      HPCP_REQUIRE(cfg.log2_elems >= 4 && cfg.log2_elems <= 32, "-p must be in [4,32]");
      return run_reduce_scatter(cfg);
    }
    HPCP_REQUIRE(cfg.algo == "ring" || cfg.algo == "ring-unfused" || cfg.algo == "ring-rsag",
                 "unknown --algo " + cfg.algo);
    HPCP_REQUIRE(cfg.log2_elems >= 4 && cfg.log2_elems <= 32, "-p must be in [4,32]");
    HPCP_REQUIRE(cfg.slots == 0 || cfg.slots == 2, "--slots must be 2 (or omitted)");
    HPCP_REQUIRE(cfg.algo != "ring-rsag" || (cfg.slots == 0 && !cfg.pull),
                 "--slots 2 and --pull are variants of --algo ring, not of ring-rsag");
    if (elem_type_is_pair(cfg.type) && !cfg.op_given) cfg.op = ReduceOp::kMaxLoc;
    HPCP_REQUIRE(cfg.op == ReduceOp::kSum || !cfg.use_collective || cfg.coll != "nvls",
                 std::string("--coll nvls is sum-only: --op ") + reduce_op_name(cfg.op) + " needs --coll twoshot or auto");
    HPCP_REQUIRE(reduce_op_takes(cfg.op, cfg.type),
                 reduce_op_type_error(cfg.op, cfg.type) +
                     (elem_type_is_pair(cfg.type) || reduce_op_on_pairs(cfg.op)
                          ? " (pass --type or run a typed binary such as allreduce.float_int)"
                          : " (pass --type or run a typed binary such as allreduce.int)"));

    if (cfg.cpu) return run_on_host(cfg);
    const int ndev = visible_device_count();
    if (ndev == 0) {
      std::cerr << "Error: No devices" << std::endl;
      return 1;
    }
    if (cfg.ranks <= 0) cfg.ranks = ndev;
    if (cfg.ranks < 2) {
      std::cerr << "Error: Set ranks to an integer >= 2 (the reference requires an even integer >= 4)"
                << std::endl;
      return 1;
    }
    const int P = cfg.ranks;
    std::vector<int> devices;
    for (int r = 0; r < P; ++r) devices.push_back(primary_device(r, P, ndev));
    const int ranks_per_dev = (P + ndev - 1) / ndev;
    if (ranks_per_dev > 1 && cfg.ctas == 0)  // co-residency of spinning kernels sharing a GPU
      cfg.ctas = std::max(1, device_sm_count(devices[0]) * 2 / ranks_per_dev);

    NodeMemory mem(devices);
    sh.mem = &mem;
    sh.n = size_t{1} << cfg.log2_elems;
    const size_t esz = elem_size(cfg.type), lanes = 16 / esz;
    const bool rsag = cfg.algo == "ring-rsag" && !cfg.use_collective;
    if ((cfg.use_collective || rsag) && sh.n % (lanes * static_cast<size_t>(P)) != 0)
      sh.n = (sh.n / (lanes * P) + 1) * (lanes * P);  // pad so that every rank owns a 16-byte aligned slice
    else if (sh.n % lanes != 0)
      sh.n = (sh.n / lanes + 1) * lanes;
    const size_t bytes = sh.n * esz;
    // ring-rsag: one arrival word per chunk of a segment
    sh.n_chunks = ring_num_chunks(rsag ? sh.n / P : sh.n, cfg.chunk_elems, elem_size(cfg.type));
    sh.pad_extra = sh.n_chunks * (cfg.slots == 2 ? 2 : 1);
    sh.epoch_advance = static_cast<uint32_t>(rsag ? rsag_epoch_advance(kRsAgAllreduce, P) : P);
    sh.pads = mem.alloc_pads(sh.pad_extra);

    if (cfg.use_collective) {
      bool want_nvls = cfg.coll == "nvls";
      if (cfg.coll == "auto") {
        // int: two-shot (128-bit peer loads for every type) — multimem.ld_reduce has no vector form for .s32;
        // float: in-switch reduction where multicast exists.
        want_nvls = ranks_per_dev == 1 && cfg.kind == AllocKind::kDevice && cfg.type == ElemType::kFloat;
        for (int d : devices) want_nvls = want_nvls && NodeMemory::multicast_supported(d);
        if (cfg.op != ReduceOp::kSum) {
          want_nvls = false;
          std::cout << "# -a --op " << reduce_op_name(cfg.op) << ": NVLS reduces sums only; using two-shot P2P"
                    << std::endl;
        }
      }
      if (want_nvls) {
        try {
          sh.mc_va = mem.alloc_multicast(bytes);
          sh.mc_vc = mem.alloc_multicast(bytes);
          sh.nvls = true;
        } catch (const std::exception& e) {
          if (cfg.coll == "nvls") throw;
          std::cerr << "# NVLS unavailable (" << e.what() << "); using two-shot P2P" << std::endl;
        }
      }
    }
    // `map` variant: the kernels' arrays are the device-resident mapped copies; the host arrays live next to them.
    const bool mapped_copy = cfg.kind == AllocKind::kMapped && !cfg.map_alias;
    const AllocKind array_kind = mapped_copy ? AllocKind::kDevice : cfg.kind;
    if (mapped_copy) {
      sh.host_va.resize(P);
      sh.host_vc.resize(P);
      for (int r = 0; r < P; ++r) {
        sh.host_va[r] = std::malloc(bytes);   // never read on the host: map(alloc) copies nothing
        sh.host_vc[r] = std::malloc(bytes);
        HPCP_REQUIRE(sh.host_va[r] != nullptr && sh.host_vc[r] != nullptr, "host allocation failed");
      }
    }
    if (!sh.nvls) {
      sh.va = mem.alloc(bytes, array_kind);
      sh.vc = mem.alloc(bytes, array_kind);
    }
    if (!cfg.use_collective) {
      if (cfg.algo == "ring")
        sh.slots = mem.alloc(bytes * static_cast<size_t>(cfg.slots == 2 ? 2 : P - 1), array_kind, /*zero=*/false);
      else if (rsag)
        sh.slots = mem.alloc(bytes / P * (P - 1), array_kind, /*zero=*/false);
      else
        sh.vb = mem.alloc(bytes, array_kind);
    }

    run_ranks(P, [&](RankCtx& ctx) { rank_main(ctx, sh); });
    for (void* h : sh.host_va) std::free(h);   // `target exit data map(delete)` + free (:168-170)
    for (void* h : sh.host_vc) std::free(h);

    // Reporting: the number the reference computes and drops.
    const std::string algo_name =
        cfg.use_collective ? (sh.nvls ? "nvls" : "twoshot") : cfg.algo;
    // Per-rank bytes sent over NVLink: faithful ring (P-1)*N; bandwidth-optimal collectives (P-1)/P*N; the
    // reduce-scatter + all-gather ring 2(P-1)/P*N.
    const double sent = cfg.use_collective ? static_cast<double>(bytes) * (P - 1) / P
                        : rsag             ? 2.0 * static_cast<double>(bytes) * (P - 1) / P
                                           : static_cast<double>(bytes) * (P - 1);
    const double gbps = sent / (sh.best_ms * 1e-3) * 1e-9;
    std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << sh.best_ms << " ms | "
              << algo_name << " " << elem_type_name(cfg.type) << " " << alloc_kind_name(cfg.kind)
              << " P=" << P << " N=2^" << cfg.log2_elems
              << (cfg.op != ReduceOp::kSum ? std::string(" op=") + reduce_op_name(cfg.op) : std::string()) << " | " << gbps
              << " GB/s sent per rank (" << gbps / 450.0 * 100.0 << "% of the 450 GB/s NVLink 4 nominal per direction)"
              << std::endl;
    if (!cfg.json_path.empty()) {
      FILE* f = std::fopen(cfg.json_path.c_str(), "a");
      if (f) {
        std::fprintf(f,
                     "{\"pattern\":\"allreduce\",\"algo\":\"%s\",\"type\":\"%s\",\"alloc\":\"%s\","
                     "\"ranks\":%d,\"elements\":%zu,\"ms\":%.6f,\"GBps_sent_per_rank\":%.3f,"
                     "\"mismatches\":%llu%s}\n",
                     algo_name.c_str(), elem_type_name(cfg.type), alloc_kind_name(cfg.kind), P, sh.n,
                     sh.best_ms, gbps, sh.total_bad, op_json(cfg.op).c_str());
        std::fclose(f);
      }
    }

    if (sh.nvls) {
      mem.free_multicast(sh.mc_va);
      mem.free_multicast(sh.mc_vc);
    } else {
      mem.free(sh.va);
      mem.free(sh.vc);
    }
    mem.free(sh.slots);
    mem.free(sh.vb);
    mem.free(sh.pads);
    return sh.total_bad == 0 ? 0 : 1;
  } catch (const std::exception& e) {
    std::cerr << "Error: " << e.what() << std::endl;
    return 1;
  }
}
