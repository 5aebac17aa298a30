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
// Additions: the elapsed time the reference computes but never prints
// (allreduce-mpi-sycl.cpp:185-190) is printed as max over ranks, with bus GB/s.
//
// Algorithms (--algo):
//   ring          fused K-ring: all P-1 exchanges + P accumulations in one launch/rank
//   ring-unfused  same data movement as the reference with separate kernels:
//                 rendezvous put kernel, then Accumulate kernel, per step (VA/VB swap)
//   (with -a)     nvls when NVSwitch multicast is available, else two-shot P2P;
//                 force with --coll nvls|twoshot
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
#include "devices.hpp"

namespace {

using namespace hpcp;


struct Config {
  int ranks = 0;
  int log2_elems = 25;
  bool use_collective = false;
  AllocKind kind = AllocKind::kDevice;
  ElemType type = ElemType::kFloat;
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
               " --type T   element type: float int uint double long ulong short ushort uchar (default float, or binary-name suffix)\n"
               " --algo ring|ring-unfused   fused persistent ring kernel (default) or\n"
               "                            separate put + accumulate kernels per step\n"
               " --coll auto|nvls|twoshot   collective used with -a\n"
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
  SymmetricBuffer va, vb, vc, slots, pads;
  MulticastBuffer mc_va, mc_vc;
  std::vector<void*> host_va, host_vc;  // -R: the host arrays whose mapped copies are va / vc
  bool nvls = false;
  double best_ms = 0;
  unsigned long long total_bad = 0;
};

double first_element_as_double(const void* p, ElemType t) {
  switch (t) {
    case ElemType::kFloat: return *static_cast<const float*>(p);
    case ElemType::kInt: return *static_cast<const int*>(p);
    case ElemType::kUInt: return *static_cast<const unsigned int*>(p);
    case ElemType::kDouble: return *static_cast<const double*>(p);
    case ElemType::kLong: return static_cast<double>(*static_cast<const long long*>(p));
    case ElemType::kULong: return static_cast<double>(*static_cast<const unsigned long long*>(p));
    case ElemType::kShort: return *static_cast<const short*>(p);
    case ElemType::kUShort: return *static_cast<const unsigned short*>(p);
    case ElemType::kUChar: return *static_cast<const unsigned char*>(p);
  }
  return 0;
}

template <typename T>
unsigned long long count_mismatch_typed(const void* p, size_t n, double expected) {
  const T* v = static_cast<const T*>(p);
  unsigned long long bad = 0;
  for (size_t i = 0; i < n; ++i) {
    const double d = static_cast<double>(v[i]) - expected;
    bad += !(d < 1e-6 && d > -1e-6);
  }
  return bad;
}
unsigned long long count_mismatch_on_host(const void* p, size_t n, double expected, ElemType t) {
  switch (t) {
    case ElemType::kFloat: return count_mismatch_typed<float>(p, n, expected);
    case ElemType::kInt: return count_mismatch_typed<int>(p, n, expected);
    case ElemType::kUInt: return count_mismatch_typed<unsigned int>(p, n, expected);
    case ElemType::kDouble: return count_mismatch_typed<double>(p, n, expected);
    case ElemType::kLong: return count_mismatch_typed<long long>(p, n, expected);
    case ElemType::kULong: return count_mismatch_typed<unsigned long long>(p, n, expected);
    case ElemType::kShort: return count_mismatch_typed<short>(p, n, expected);
    case ElemType::kUShort: return count_mismatch_typed<unsigned short>(p, n, expected);
    case ElemType::kUChar: return count_mismatch_typed<unsigned char>(p, n, expected);
  }
  return n;
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
      a.epoch_base = replay ? ring_epoch - static_cast<uint32_t>(P) : ring_epoch;
      a.timeout_ns = cfg.timeout_ns;
      a.status = status;
      a.n_slots = cfg.slots;
      if (cfg.pull) {  // receiver-driven: load from the left neighbour instead of being stored into
        a.pull = true;
        a.va_left = sh.va.ptr[left];
        a.slots_left = sh.slots.ptr[left];
      }
      if (cfg.slots == 2) {  // ack words follow the arrival words on every pad
        a.ack_local = my_pad + kPadWords + sh.n_chunks;
        a.ack_left = pad_of(sh, left) + kPadWords + sh.n_chunks;
      }
      if (!replay) ring_epoch += static_cast<uint32_t>(P);
      launch_ring_allreduce(a, cfg.type, cfg.ctas, dev, stream);
    } else {  // ring-unfused: the reference's step structure with separate kernels
      HPCP_REQUIRE(!replay, "--profile-relaunch supports the one-launch algorithms only");
      void* cur = va;
      void* other = sh.vb.ptr[me];
      void* right_cur = sh.va.ptr[right];     // what the right neighbour currently calls VA
      void* right_other = sh.vb.ptr[right];   // ... and VB (where my block must land)
      launch_accumulate(cur, vc, sh.n, cfg.type, stream);
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
        launch_accumulate(cur, vc, sh.n, cfg.type, stream);
      }
    }

  };

  for (int it = 0; it < cfg.warmup + cfg.iters; ++it) {
    NvtxRange iter_range(it < cfg.warmup ? "allreduce warm-up" : "allreduce timed");
    // (Re-)initialise outside the timed region: VA = VB = rank, VC = 0.
    launch_init3(va, cfg.algo == "ring-unfused" && !cfg.use_collective ? sh.vb.ptr[me] : nullptr, vc,
                 sh.n, me, me, 0, cfg.type, stream);
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

  // Verify: every element of VC equals P(P-1)/2.
  unsigned long long bad = 0;
  const bool mapped_copy = !sh.host_vc.empty();
  if (mapped_copy) {
    // `#pragma omp target update from(VC[:n])` (allreduce-map-mpi-omp-offload.cpp:159), then the host checks its
    // own array (:163-164) and prints "<rank> <VC[0]>" (:161).
    HPCP_CUDA(cudaMemcpyAsync(sh.host_vc[me], vc, sh.n * esz, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    bad = count_mismatch_on_host(sh.host_vc[me], sh.n, 0.5 * P * (P - 1), cfg.type);
  } else {
    unsigned long long* count = nullptr;
    HPCP_CUDA(cudaMalloc(&count, sizeof *count));
    HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
    launch_count_mismatch(vc, sh.n, 0.5 * P * (P - 1), cfg.type, count, stream);
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
template <typename T>
int run_on_host_typed(const Config& cfg) {
  const int P = cfg.ranks > 0 ? cfg.ranks : 4;
  const size_t n = size_t{1} << cfg.log2_elems;
  std::vector<std::vector<T>> va(P), vb(P), vc(P);
  double elapsed_ms = 0;
  unsigned long long total_bad = 0;
  run_ranks(P, [&](RankCtx& ctx) {
    const int me = ctx.rank, right = (me + 1) % P;
    va[me].assign(n, static_cast<T>(me));
    vb[me].assign(n, static_cast<T>(me));
    vc[me].assign(n, static_cast<T>(0));
    ctx.barrier();
    const auto t0 = std::chrono::steady_clock::now();
    if (cfg.use_collective) {
      for (int r = 0; r < P; ++r)
        for (size_t i = 0; i < n; ++i) vc[me][i] += va[r][i];
    } else {
      for (size_t i = 0; i < n; ++i) vc[me][i] += va[me][i];
      for (int s = 1; s < P; ++s) {
        std::memcpy(vb[right].data(), va[me].data(), n * sizeof(T));  // "send right"
        ctx.barrier();                                                 // everybody received
        va[me].swap(vb[me]);
        ctx.barrier();                                                 // nobody still reads the old VA
        for (size_t i = 0; i < n; ++i) vc[me][i] += va[me][i];
      }
    }
    const double ms =
        std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const double t = ctx.max(ms);
    const T want = static_cast<T>(P * (P - 1) / 2);
    unsigned long long bad = 0;
    for (size_t i = 0; i < n; ++i) bad += std::abs(static_cast<double>(vc[me][i]) - static_cast<double>(want)) >= 1e-6;
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
            << (cfg.use_collective ? "collective" : "ring") << " " << elem_type_name(cfg.type)
            << " host-threads P=" << P << " N=2^" << cfg.log2_elems << " arrays=" << alloc_kind_name(cfg.kind)
            << " (host vectors in this mode)" << std::endl;
  if (!cfg.json_path.empty()) {  // same row shape as the GPU path; the algo name marks the plumbing run
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      const size_t n = size_t{1} << cfg.log2_elems;
      const double sent = cfg.use_collective ? 0.0 : static_cast<double>(P - 1) * n * sizeof(T);
      std::fprintf(f,
                   "{\"pattern\":\"allreduce\",\"algo\":\"%s\",\"type\":\"%s\",\"alloc\":\"host-vectors\","
                   "\"ranks\":%d,\"elements\":%zu,\"ms\":%.6f,\"GBps_sent_per_rank\":%.3f,\"mismatches\":%llu}\n",
                   cfg.use_collective ? "host-collective" : "host-ring", elem_type_name(cfg.type), P, n, elapsed_ms,
                   elapsed_ms > 0 ? sent / (elapsed_ms * 1e6) : 0.0, total_bad);
      std::fclose(f);
    }
  }
  return total_bad == 0 ? 0 : 1;
}

int run_on_host(const Config& cfg) {
  switch (cfg.type) {
    case ElemType::kFloat: return run_on_host_typed<float>(cfg);
    case ElemType::kInt: return run_on_host_typed<int>(cfg);
    case ElemType::kUInt: return run_on_host_typed<unsigned int>(cfg);
    case ElemType::kDouble: return run_on_host_typed<double>(cfg);
    case ElemType::kLong: return run_on_host_typed<long long>(cfg);
    case ElemType::kULong: return run_on_host_typed<unsigned long long>(cfg);
    case ElemType::kShort: return run_on_host_typed<short>(cfg);
    case ElemType::kUShort: return run_on_host_typed<unsigned short>(cfg);
    case ElemType::kUChar: return run_on_host_typed<unsigned char>(cfg);
  }
  return 1;
}
}  // namespace

int main(int argc, char** argv) {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  try {
    Shared sh;
    Config& cfg = sh.cfg;
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
                                       {"help", no_argument, nullptr, 'h'},
                                       {nullptr, 0, nullptr, 0}};
    int opt;
    while ((opt = getopt_long(argc, argv, "haHDSRp:n:", long_opts, nullptr)) != -1) {
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
        case 10: cfg.slots = std::atoi(optarg); break;
        case 11: cfg.pull = true; break;
        default: print_help(); return 1;
      }
    }
    HPCP_REQUIRE(cfg.algo == "ring" || cfg.algo == "ring-unfused", "unknown --algo " + cfg.algo);
    HPCP_REQUIRE(cfg.log2_elems >= 4 && cfg.log2_elems <= 32, "-p must be in [4,32]");
    HPCP_REQUIRE(cfg.slots == 0 || cfg.slots == 2, "--slots must be 2 (or omitted)");

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
    if (cfg.use_collective && sh.n % (lanes * static_cast<size_t>(P)) != 0)
      sh.n = (sh.n / (lanes * P) + 1) * (lanes * P);  // pad so that every rank owns a 16-byte aligned slice
    else if (sh.n % lanes != 0)
      sh.n = (sh.n / lanes + 1) * lanes;
    const size_t bytes = sh.n * esz;
    sh.n_chunks = ring_num_chunks(sh.n, cfg.chunk_elems, elem_size(cfg.type));
    sh.pad_extra = sh.n_chunks * (cfg.slots == 2 ? 2 : 1);
    sh.pads = mem.alloc_pads(sh.pad_extra);

    if (cfg.use_collective) {
      bool want_nvls = cfg.coll == "nvls";
      if (cfg.coll == "auto") {
        // int: two-shot (128-bit peer loads for every type) — multimem.ld_reduce has no vector form for .s32;
        // float: in-switch reduction where multicast exists.
        want_nvls = ranks_per_dev == 1 && cfg.kind == AllocKind::kDevice && cfg.type == ElemType::kFloat;
        for (int d : devices) want_nvls = want_nvls && NodeMemory::multicast_supported(d);
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
      else
        sh.vb = mem.alloc(bytes, array_kind);
    }

    run_ranks(P, [&](RankCtx& ctx) { rank_main(ctx, sh); });
    for (void* h : sh.host_va) std::free(h);   // `target exit data map(delete)` + free (:168-170)
    for (void* h : sh.host_vc) std::free(h);

    // Reporting: the number the reference computes and drops.
    const std::string algo_name =
        cfg.use_collective ? (sh.nvls ? "nvls" : "twoshot") : cfg.algo;
    // Per-rank bytes sent over NVLink: faithful ring (P-1)*N; bandwidth-optimal collectives (P-1)/P*N.
    const double sent = cfg.use_collective ? static_cast<double>(bytes) * (P - 1) / P
                                           : static_cast<double>(bytes) * (P - 1);
    const double gbps = sent / (sh.best_ms * 1e-3) * 1e-9;
    std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << sh.best_ms << " ms | "
              << algo_name << " " << elem_type_name(cfg.type) << " " << alloc_kind_name(cfg.kind)
              << " P=" << P << " N=2^" << cfg.log2_elems << " | " << gbps
              << " GB/s sent per rank (" << gbps / 450.0 * 100.0 << "% of the 450 GB/s NVLink 4 nominal per direction)"
              << std::endl;
    if (!cfg.json_path.empty()) {
      FILE* f = std::fopen(cfg.json_path.c_str(), "a");
      if (f) {
        std::fprintf(f,
                     "{\"pattern\":\"allreduce\",\"algo\":\"%s\",\"type\":\"%s\",\"alloc\":\"%s\","
                     "\"ranks\":%d,\"elements\":%zu,\"ms\":%.6f,\"GBps_sent_per_rank\":%.3f,"
                     "\"mismatches\":%llu}\n",
                     algo_name.c_str(), elem_type_name(cfg.type), alloc_kind_name(cfg.kind), P, sh.n,
                     sh.best_ms, gbps, sh.total_bad);
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
