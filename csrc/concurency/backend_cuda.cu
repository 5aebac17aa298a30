// CUDA backend of the concurrency benchmark (H100).
//
// Same question as the reference's SYCL and OpenMP-offload backends
// (concurency/bench_sycl.cpp:19-139, bench_omp.cpp:21-137) — do independent
// commands overlap? — asked through every submission idiom the CUDA stack has,
// all selectable at run time:
//   serial        one stream, host sync after every command (the baseline)
//   in_order      N in-order streams, command i -> stream i % N     (↔ SYCL in_order queues)
//   out_of_order  ONE CUDA graph whose nodes have no edges; the runtime finds
//                 the parallelism                                   (↔ SYCL out-of-order queue)
//   host_threads  one host thread + stream per command              (↔ OpenMP host_threads)
//   nowait        one thread, async launches on non-blocking streams, event
//                 join on a master stream                           (↔ OpenMP target nowait + taskwait)
//   fused         the whole group as ONE persistent sm_90a kernel: CTAs split
//                 between FMA/triad math and TMA copy engines        (new — the product)
// Memory letters: M pageable, H pinned, D device, S managed, P peer GPU (NVLink).
#include <atomic>
#include <chrono>
#include <cstring>
#include <exception>
#include <iostream>
#include <limits>
#include <numeric>
#include <stdexcept>
#include <thread>

#include "../common/cuda_check.h"
#include "../common/peer_mem.h"
#include "../kernels/api.h"
#include "bench.hpp"
#include "driver.hpp"

namespace hpcp {
namespace con {

namespace {

using Clock = std::chrono::steady_clock;
long elapsed_us(Clock::time_point a, Clock::time_point b) {
  return static_cast<long>(std::chrono::duration_cast<std::chrono::microseconds>(b - a).count());
}

struct DevCommand {
  std::string name;
  size_t n = 0;
  size_t tripcount = 0;
  int device = 0;
  // copies
  void* src = nullptr;
  void* dst = nullptr;
  AllocKind src_kind = AllocKind::kDevice, dst_kind = AllocKind::kDevice;
  // compute
  float* a = nullptr;
  float* b = nullptr;
  float* c = nullptr;

  bool is_copy() const { return name.size() == 2; }
  size_t bytes() const { return n * sizeof(float); }

  void submit(cudaStream_t s) const {
    if (name == "C") {
      launch_busy_wait(a, n, tripcount, s);
    } else if (name == "T") {
      // HPCP_T_CLUSTER=2: thread-block clusters of two CTAs sharing the B tile via TMA multicast.
      static const int cluster = [] {
        const char* e = std::getenv("HPCP_T_CLUSTER");
        return (e != nullptr && std::atoi(e) == 2) ? 2 : 1;
      }();
      launch_tc_busy(b, a, static_cast<int>(n), static_cast<uint32_t>(tripcount), s, cluster);
    } else if (name == "A") {
      TriadPutArgs t;
      t.a_local = a;
      t.b = b;
      t.c = c;
      t.s = 3.0f;
      t.n = n & ~static_cast<size_t>(3);  // the triad covers whole 16-byte vectors; fewer than 4 elements is no work
      if (t.n != 0) launch_triad_put(t, CopyEngine::kLdSt, CopyTuning{}, SyncOps{}, nullptr, 0, device, s);
    } else {
      HPCP_CUDA(cudaMemcpyAsync(dst, src, bytes(), cudaMemcpyDefault, s));
    }
  }
};

class CudaBackend final : public Backend {
 public:
  CudaBackend(int device, int peer) : device_(device), peer_(peer) {
    HPCP_CUDA(cudaSetDevice(device_));
    if (peer_ >= 0) enable_peer_access({device_, peer_});
  }

  std::string name() const override {
    cudaDeviceProp p{};
    (void)cudaGetDeviceProperties(&p, device_);
    return std::string("cuda:") + std::to_string(device_) + " (" + p.name + ")";
  }
  std::vector<std::string> modes() const override {
    return {"in_order", "out_of_order", "host_threads", "nowait", "fused"};
  }
  std::string memory_letters() const override { return peer_ >= 0 ? "MDHSP" : "MDHS"; }
  std::string compute_letters() const override { return "CAT"; }

  BenchResult run(const BenchRequest& req) override {
    HPCP_CUDA(cudaSetDevice(device_));
    std::vector<DevCommand> cmds = build(req);
    BenchResult res;
    try {
      if (req.mode == "serial")
        res = run_serial(req, cmds);
      else if (req.mode == "in_order")
        res = run_streams(req, cmds, /*nonblocking_join=*/false);
      else if (req.mode == "nowait")
        res = run_streams(req, cmds, /*nonblocking_join=*/true);
      else if (req.mode == "out_of_order")
        res = run_graph(req, cmds);
      else if (req.mode == "host_threads")
        res = run_threads(req, cmds);
      else if (req.mode == "fused")
        res = run_fused(req, cmds);
      else
        throw std::runtime_error("cuda backend: unknown mode '" + req.mode + "'");
    } catch (...) {
      destroy(cmds);
      throw;
    }
    destroy(cmds);
    return res;
  }

 private:
  int device_;
  int peer_;

  void* make_buffer(char letter, size_t bytes, AllocKind* kind_out) const {
    const AllocKind kind = letter == 'P' ? AllocKind::kDevice : alloc_kind_from_letter(letter);
    *kind_out = kind;
    return alloc_bytes(bytes, kind, letter == 'P' ? peer_ : device_, /*zero=*/true);
  }

  std::vector<DevCommand> build(const BenchRequest& req) const {
    std::vector<DevCommand> cmds;
    try {
      build_into(req, cmds);
    } catch (...) {
      destroy(cmds);  // a failed allocation must not leak the buffers of the commands before it
      throw;
    }
    return cmds;
  }

  void build_into(const BenchRequest& req, std::vector<DevCommand>& cmds) const {
    for (const auto& name : req.commands) {
      cmds.emplace_back();
      DevCommand& c = cmds.back();
      c.name = name;
      c.device = device_;
      c.n = require_param(req, "globalsize_" + name);
      if (name == "C") {
        c.tripcount = require_param(req, "tripcount_C");
        c.a = static_cast<float*>(alloc_bytes(c.n * sizeof(float), AllocKind::kDevice, device_, true));
      } else if (name == "T") {
        // n = CTAs (one 128x256 accumulator tile each); b = bf16 operands A|B; a = fp32 results.
        // HPCP_T_OUT=P puts the accumulator tiles into the PEER GPU: the epilogue stores
        // straight over NVLink, i.e. tensor-core tile compute -> P2P put in one kernel.
        c.tripcount = require_param(req, "tripcount_T");
        const char* t_out = std::getenv("HPCP_T_OUT");
        const int out_dev = (t_out != nullptr && t_out[0] == 'P' && peer_ >= 0) ? peer_ : device_;
        c.a = static_cast<float*>(alloc_bytes(c.n * tc_busy_out_elems_per_cta() * sizeof(float),
                                              AllocKind::kDevice, out_dev, true));
        c.b = static_cast<float*>(alloc_bytes(tc_busy_operand_bytes(), AllocKind::kDevice, device_, true));
        launch_tc_fill_operands(c.b, nullptr);
      } else if (name == "A") {
        c.a = static_cast<float*>(alloc_bytes(c.bytes(), AllocKind::kDevice, device_, true));
        c.b = static_cast<float*>(alloc_bytes(c.bytes(), AllocKind::kDevice, device_, true));
        c.c = static_cast<float*>(alloc_bytes(c.bytes(), AllocKind::kDevice, device_, true));
      } else {
        c.src = make_buffer(name[0], c.bytes(), &c.src_kind);
        c.dst = make_buffer(name[1], c.bytes(), &c.dst_kind);
      }
    }
    HPCP_CUDA(cudaDeviceSynchronize());
  }

  void destroy(std::vector<DevCommand>& cmds) const {
    (void)cudaDeviceSynchronize();
    for (auto& c : cmds) {
      free_bytes(c.a, AllocKind::kDevice);
      free_bytes(c.b, AllocKind::kDevice);
      free_bytes(c.c, AllocKind::kDevice);
      if (c.is_copy()) {
        free_bytes(c.src, c.src_kind);
        free_bytes(c.dst, c.dst_kind);
      }
    }
    cmds.clear();
  }

  static void note_rep(const BenchRequest& req, int r, long t) {
    if (req.verbose) std::cout << "#repetition " << r << ": " << t << " us" << std::endl;
  }

  // ---- serial ------------------------------------------------------------
  BenchResult run_serial(const BenchRequest& req, const std::vector<DevCommand>& cmds) const {
    const size_t nc = cmds.size();
    if (req.verbose) std::cout << "#n_queues used: 1" << std::endl;
    cudaStream_t s;
    HPCP_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    std::vector<cudaEvent_t> ev(2 * nc);
    if (req.enable_profiling)
      for (auto& e : ev) HPCP_CUDA(cudaEventCreate(&e));

    BenchResult res;
    res.total_us = std::numeric_limits<long>::max();
    res.per_command_us.assign(nc, std::numeric_limits<long>::max());
    if (req.enable_profiling) res.device_us.assign(nc, std::numeric_limits<double>::max());
    for (int r = 0; r < req.n_repetitions; ++r) {
      const auto t0 = Clock::now();
      for (size_t i = 0; i < nc; ++i) {
        const auto s0 = Clock::now();
        if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(ev[2 * i], s));
        cmds[i].submit(s);
        if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(ev[2 * i + 1], s));
        HPCP_CUDA(cudaStreamSynchronize(s));
        res.per_command_us[i] = std::min(res.per_command_us[i], elapsed_us(s0, Clock::now()));
        if (req.enable_profiling) {
          float ms = 0;
          HPCP_CUDA(cudaEventElapsedTime(&ms, ev[2 * i], ev[2 * i + 1]));
          res.device_us[i] = std::min(res.device_us[i], 1e3 * static_cast<double>(ms));
        }
      }
      const long t = elapsed_us(t0, Clock::now());
      note_rep(req, r, t);
      res.total_us = std::min(res.total_us, t);
    }
    res.total_us = std::min(
        res.total_us, std::accumulate(res.per_command_us.begin(), res.per_command_us.end(), 0L));
    if (req.enable_profiling)
      for (auto& e : ev) (void)cudaEventDestroy(e);
    (void)cudaStreamDestroy(s);
    return res;
  }

  // ---- in_order / nowait ----------------------------------------------------
  BenchResult run_streams(const BenchRequest& req, const std::vector<DevCommand>& cmds,
                          bool nonblocking_join) const {
    const size_t nc = cmds.size();
    int nq = req.n_queues == -1 ? static_cast<int>(nc) : req.n_queues;
    nq = std::max(nq, 1);
    if (req.verbose) std::cout << "#n_queues used: " << nq << std::endl;
    std::vector<cudaStream_t> qs(nq);
    for (auto& q : qs) HPCP_CUDA(cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
    cudaStream_t master;
    HPCP_CUDA(cudaStreamCreateWithFlags(&master, cudaStreamNonBlocking));
    std::vector<cudaEvent_t> done(nq);
    for (auto& e : done) HPCP_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    cudaEvent_t g0, g1;
    HPCP_CUDA(cudaEventCreate(&g0));
    HPCP_CUDA(cudaEventCreate(&g1));
    const bool joined = nonblocking_join || req.enable_profiling;

    BenchResult res;
    res.total_us = std::numeric_limits<long>::max();
    double dev_best = std::numeric_limits<double>::max();
    for (int r = 0; r < req.n_repetitions; ++r) {
      const auto t0 = Clock::now();
      if (req.enable_profiling) {
        HPCP_CUDA(cudaEventRecord(g0, master));
        for (auto& q : qs) HPCP_CUDA(cudaStreamWaitEvent(q, g0, 0));
      }
      for (size_t i = 0; i < nc; ++i) cmds[i].submit(qs[i % nq]);
      if (joined) {
        // "taskwait": the master stream joins every queue on the device; one host sync.
        for (int q = 0; q < nq; ++q) {
          HPCP_CUDA(cudaEventRecord(done[q], qs[q]));
          HPCP_CUDA(cudaStreamWaitEvent(master, done[q], 0));
        }
        if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(g1, master));
        HPCP_CUDA(cudaStreamSynchronize(master));
      } else {
        for (auto& q : qs) HPCP_CUDA(cudaStreamSynchronize(q));
      }
      const long t = elapsed_us(t0, Clock::now());
      note_rep(req, r, t);
      res.total_us = std::min(res.total_us, t);
      if (req.enable_profiling) {
        float ms = 0;
        HPCP_CUDA(cudaEventElapsedTime(&ms, g0, g1));
        dev_best = std::min(dev_best, 1e3 * static_cast<double>(ms));
      }
    }
    if (req.enable_profiling) res.device_total_us = dev_best;
    (void)cudaEventDestroy(g0);
    (void)cudaEventDestroy(g1);
    for (auto& e : done) (void)cudaEventDestroy(e);
    for (auto& q : qs) (void)cudaStreamDestroy(q);
    (void)cudaStreamDestroy(master);
    return res;
  }

  // ---- out_of_order ---------------------------------------------------------
  BenchResult run_graph(const BenchRequest& req, const std::vector<DevCommand>& cmds) const {
    if (req.verbose) std::cout << "#n_queues used: 1" << std::endl;
    cudaStream_t s;
    HPCP_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    cudaGraph_t graph;
    HPCP_CUDA(cudaGraphCreate(&graph, 0));
    std::vector<cudaGraph_t> children;
    for (const auto& c : cmds) {
      cudaGraphNode_t node;
      const bool pageable = c.is_copy() && (c.src_kind == AllocKind::kPageable ||
                                            c.dst_kind == AllocKind::kPageable);
      if (pageable) {
        // Pageable copies cannot be stream-captured; add an explicit memcpy node.
        HPCP_CUDA(cudaGraphAddMemcpyNode1D(&node, graph, nullptr, 0, c.dst, c.src, c.bytes(),
                                           cudaMemcpyDefault));
      } else {
        cudaGraph_t child;
        HPCP_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
        c.submit(s);
        HPCP_CUDA(cudaStreamEndCapture(s, &child));
        HPCP_CUDA(cudaGraphAddChildGraphNode(&node, graph, nullptr, 0, child));
        children.push_back(child);
      }
    }
    cudaGraphExec_t exec;
    HPCP_CUDA(cudaGraphInstantiate(&exec, graph, 0));
    cudaEvent_t g0, g1;
    HPCP_CUDA(cudaEventCreate(&g0));
    HPCP_CUDA(cudaEventCreate(&g1));

    BenchResult res;
    res.total_us = std::numeric_limits<long>::max();
    double dev_best = std::numeric_limits<double>::max();
    for (int r = 0; r < req.n_repetitions; ++r) {
      const auto t0 = Clock::now();
      if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(g0, s));
      HPCP_CUDA(cudaGraphLaunch(exec, s));
      if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(g1, s));
      HPCP_CUDA(cudaStreamSynchronize(s));
      const long t = elapsed_us(t0, Clock::now());
      note_rep(req, r, t);
      res.total_us = std::min(res.total_us, t);
      if (req.enable_profiling) {
        float ms = 0;
        HPCP_CUDA(cudaEventElapsedTime(&ms, g0, g1));
        dev_best = std::min(dev_best, 1e3 * static_cast<double>(ms));
      }
    }
    if (req.enable_profiling) res.device_total_us = dev_best;
    (void)cudaEventDestroy(g0);
    (void)cudaEventDestroy(g1);
    (void)cudaGraphExecDestroy(exec);
    for (auto& ch : children) (void)cudaGraphDestroy(ch);
    (void)cudaGraphDestroy(graph);
    (void)cudaStreamDestroy(s);
    return res;
  }

  // ---- host_threads -------------------------------------------------------
  BenchResult run_threads(const BenchRequest& req, const std::vector<DevCommand>& cmds) const {
    const size_t nc = cmds.size();
    int nq = req.n_queues == -1 ? static_cast<int>(nc) : req.n_queues;
    nq = std::max(nq, 1);
    if (req.verbose) std::cout << "#n_queues used: " << nq << std::endl;
    std::vector<cudaStream_t> qs(nq);
    for (auto& q : qs) HPCP_CUDA(cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));

    // Persistent workers: each repetition is released by bumping `go`.
    std::atomic<int> go{0}, finished{0};
    std::atomic<bool> quit{false};
    std::vector<std::string> errors(nq);
    std::vector<std::thread> workers;
    for (int w = 0; w < nq; ++w) {
      workers.emplace_back([&, w] {
        try {
          HPCP_CUDA(cudaSetDevice(device_));
          int seen = 0;
          while (true) {
            while (go.load(std::memory_order_acquire) == seen && !quit.load()) {
            }
            if (quit.load()) return;
            ++seen;
            for (size_t i = w; i < nc; i += nq) cmds[i].submit(qs[w]);
            HPCP_CUDA(cudaStreamSynchronize(qs[w]));
            finished.fetch_add(1, std::memory_order_release);
          }
        } catch (const std::exception& e) {
          errors[w] = e.what();
          finished.fetch_add(1 << 16, std::memory_order_release);
        }
      });
    }

    BenchResult res;
    res.total_us = std::numeric_limits<long>::max();
    bool failed = false;
    for (int r = 0; r < req.n_repetitions && !failed; ++r) {
      finished.store(0);
      const auto t0 = Clock::now();
      go.fetch_add(1, std::memory_order_release);
      while (true) {
        const int f = finished.load(std::memory_order_acquire);
        if (f >= (1 << 16)) {
          failed = true;
          break;
        }
        if (f == nq) break;
      }
      const long t = elapsed_us(t0, Clock::now());
      note_rep(req, r, t);
      res.total_us = std::min(res.total_us, t);
    }
    quit.store(true);
    for (auto& t : workers) t.join();
    for (auto& q : qs) (void)cudaStreamDestroy(q);
    for (const auto& e : errors)
      if (!e.empty()) throw std::runtime_error("host_threads worker failed: " + e);
    return res;
  }

  // ---- fused ----------------------------------------------------------------
  BenchResult run_fused(const BenchRequest& req, const std::vector<DevCommand>& cmds) const {
    if (req.verbose) std::cout << "#n_queues used: 1" << std::endl;
    std::vector<FusedCommand> fused;
    std::vector<const DevCommand*> side;  // launched alongside the fused kernel, one stream each
    // PCIe traffic driven from the SMs (zero-copy TMA / ld-st on pinned memory) can reach copy-engine
    // speed in ONE direction but not in both at once: with two or more host copies in the group they go
    // to the copy engines.  The same holds for NVLink when one GPU drives both directions at once (put +
    // get from the same SMs).
    int host_copies = 0, peer_copies = 0;
    for (const auto& c : cmds) {
      if (!c.is_copy()) continue;
      if (c.src_kind == AllocKind::kPinned || c.dst_kind == AllocKind::kPinned) ++host_copies;
      if (c.name[0] == 'P' || c.name[1] == 'P') ++peer_copies;
    }
    const bool host_copies_on_ce = host_copies >= 2 && std::getenv("HPCP_FUSED_HOST_ZERO_COPY") == nullptr;
    const bool peer_copies_on_ce = peer_copies >= 2 && std::getenv("HPCP_FUSED_PEER_IN_KERNEL") == nullptr;
    for (const auto& c : cmds) {
      FusedCommand f;
      if (c.name == "C") {
        f.kind = FusedKind::kBusy;
        f.n = c.n;
        f.tripcount = c.tripcount;
        f.a = c.a;
      } else if (c.name == "A") {
        f.kind = FusedKind::kTriad;
        f.n = c.n;
        f.a = c.a;
        f.b = c.b;
        f.c = c.c;
      } else if (c.name == "T") {
        side.push_back(&c);  // tensor-core tile loop: its own (smem-hungry) kernel
        continue;
      } else if (c.src_kind == AllocKind::kPageable || c.dst_kind == AllocKind::kPageable) {
        side.push_back(&c);  // a kernel cannot dereference pageable host memory on x86 H100
        continue;
      } else if (host_copies_on_ce && (c.src_kind == AllocKind::kPinned || c.dst_kind == AllocKind::kPinned)) {
        side.push_back(&c);
        continue;
      } else if (peer_copies_on_ce && (c.name[0] == 'P' || c.name[1] == 'P')) {
        side.push_back(&c);
        continue;
      } else {
        f.kind = FusedKind::kCopy;
        f.n = c.n;
        f.dst = c.dst;
        f.src = c.src;
        // A link-bound copy needs few DMA CTAs; the SMs it does not take stay with the math
        // (PCIe: 16 CTAs; NVLink: 64 CTAs; HBM<->HBM copies share the pool).
        const bool host = c.src_kind == AllocKind::kPinned || c.dst_kind == AllocKind::kPinned;
        const bool peer = c.name[0] == 'P' || c.name[1] == 'P';
        if (host) f.ctas = 16;
        else if (peer) f.ctas = 64;
      }
      fused.push_back(f);
    }
    CopyEngine engine = CopyEngine::kTma;
    if (const char* e = std::getenv("HPCP_FUSED_COPY_ENGINE"))
      if (std::string(e) == "ldst") engine = CopyEngine::kLdSt;

    cudaStream_t s;
    HPCP_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    std::vector<cudaStream_t> side_streams(side.size());
    for (auto& q : side_streams) HPCP_CUDA(cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
    cudaEvent_t g0, g1;
    HPCP_CUDA(cudaEventCreate(&g0));
    HPCP_CUDA(cudaEventCreate(&g1));
    BenchResult res;
    res.total_us = std::numeric_limits<long>::max();
    double dev_best = std::numeric_limits<double>::max();
    // A copy that touches pageable memory blocks its calling thread while the driver stages it, and it does not
    // reliably overlap a kernel enqueued by the SAME thread just before it.  Each side copy therefore gets its own host thread — the reference's
    // host_threads idiom (concurency/bench_omp.cpp:67-69) for the one thing a kernel cannot do itself: x86 H100s
    // cannot dereference pageable memory from the SMs.  HPCP_FUSED_SIDE_THREADS=0 restores the single-thread order.
    const bool side_threads = [] {
      const char* e = std::getenv("HPCP_FUSED_SIDE_THREADS");
      return e == nullptr || std::atoi(e) != 0;
    }();
    for (int r = 0; r < req.n_repetitions; ++r) {
      const auto t0 = Clock::now();
      if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(g0, s));
      // Side *kernels* (T) first: a resident-wave kernel launched earlier would otherwise hold the SMs.
      for (size_t k = 0; k < side.size(); ++k)
        if (!side[k]->is_copy()) side[k]->submit(side_streams[k]);
      std::vector<std::thread> helpers;
      std::vector<std::exception_ptr> helper_error(side.size());
      if (side_threads) {
        for (size_t k = 0; k < side.size(); ++k) {
          if (!side[k]->is_copy()) continue;
          helpers.emplace_back([&, k] {
            try {
              HPCP_CUDA(cudaSetDevice(device_));
              side[k]->submit(side_streams[k]);
              HPCP_CUDA(cudaStreamSynchronize(side_streams[k]));
            } catch (...) {
              helper_error[k] = std::current_exception();
            }
          });
        }
      }
      if (!fused.empty())
        launch_fused_bench(fused.data(), static_cast<int>(fused.size()), engine, CopyTuning{},
                           device_, s);
      if (req.enable_profiling) HPCP_CUDA(cudaEventRecord(g1, s));
      if (!side_threads)
        for (size_t k = 0; k < side.size(); ++k)
          if (side[k]->is_copy()) side[k]->submit(side_streams[k]);
      HPCP_CUDA(cudaStreamSynchronize(s));
      for (auto& t : helpers) t.join();
      for (auto& e : helper_error)
        if (e) std::rethrow_exception(e);
      for (auto& q : side_streams) HPCP_CUDA(cudaStreamSynchronize(q));
      const long t = elapsed_us(t0, Clock::now());
      note_rep(req, r, t);
      res.total_us = std::min(res.total_us, t);
      if (req.enable_profiling) {
        float ms = 0;
        HPCP_CUDA(cudaEventElapsedTime(&ms, g0, g1));
        dev_best = std::min(dev_best, 1e3 * static_cast<double>(ms));
      }
    }
    if (req.enable_profiling) res.device_total_us = dev_best;
    (void)cudaEventDestroy(g0);
    (void)cudaEventDestroy(g1);
    (void)cudaStreamDestroy(s);
    for (auto& q : side_streams) (void)cudaStreamDestroy(q);
    return res;
  }
};

}  // namespace

std::unique_ptr<Backend> make_cuda_backend(std::string* why_not) {
  int n = 0;
  const cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    (void)cudaGetLastError();
    if (why_not) *why_not = e != cudaSuccess ? cudaGetErrorString(e) : "no CUDA device";
    return nullptr;
  }
  int device = 0;
  if (const char* d = std::getenv("HPCP_DEVICE")) device = std::atoi(d);
  if (device < 0 || device >= n) device = 0;
  // Peer GPU for the `P` letter: the next ordinal with a P2P path.
  int peer = -1;
  if (const char* p = std::getenv("HPCP_PEER_DEVICE")) {
    peer = std::atoi(p);
  } else {
    for (int k = 1; k < n && peer < 0; ++k) {
      const int cand = (device + k) % n;
      int ok = 0;
      if (cudaDeviceCanAccessPeer(&ok, device, cand) == cudaSuccess && ok) peer = cand;
    }
  }
  try {
    return std::make_unique<CudaBackend>(device, peer);
  } catch (const std::exception& ex) {
    if (why_not) *why_not = ex.what();
    return nullptr;
  }
}

}  // namespace con
}  // namespace hpcp
