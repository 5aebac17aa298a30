// peer2pear — GPU<->GPU bandwidth between rank pairs over NVLink / NVSwitch.
//
// Capability parity with p2p/peer2pear.cpp of the reference:
//   * ranks are paired (2k, 2k+1); phase 1 is unidirectional (even -> odd), phase 2
//     bidirectional (peer2pear.cpp:126-146);
//   * 10 iterations, the minimum is reported (:23,52);
//   * bandwidth = bytes * pairs / t and 2 * bytes * pairs / t, aggregated over all
//     pairs, printed by rank 0 as `<label> Unidirectional Bandwidth: X GB/s` and
//     `<label> Bidirectional Bandwidth: X GB/s` (:137-140,152-155);
//   * default message = 47 185 920 floats = 188 743 680 B (:115-116);
//   * the two upstream builds (two-sided Isend/Irecv, one-sided Put+fence under
//     -DUSE_WIN) are the run-time transports `sendrecv` and `put`; `get` is new;
//     `memcpy` (cudaMemcpyPeerAsync, copy engines) is the stock-library baseline.
// H100 design: one process, one host thread per rank (rank_runtime.h), every GPU
// peer-mapped; data is moved by hand-written sm_90a kernels (kernels/p2p.cu) and
// synchronised with release/acquire epoch words in peer memory — no MPI, no NCCL.
// Time is measured on the device (CUDA events around the rank's kernels, started
// behind an in-kernel cross-GPU barrier) and reduced with max over ranks.
// Fixes over the reference: separate send / receive buffers (upstream sends from
// and receives into the same buffer, :128,142), exact device-side verification
// (upstream: float sorted-sum, :55-63), optional size sweep 1 KiB..1 GiB.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <limits>
#include <sstream>
#include <string>
#include <vector>

#include "../common/cuda_check.h"
#include "../common/nvtx.h"
#include "../common/peer_mem.h"
#include "../common/rank_runtime.h"
#include "../common/signal_layout.h"
#include "../kernels/api.h"
#include "../kernels/payload.h"
#include "topology_core.hpp"

namespace {

using namespace hpcp;


struct Config {
  std::string label = "Tile2Tile";
  int ranks = 0;  // 0 -> all GPUs (rounded down to even)
  std::string transport = "put";
  std::string engine = "tma";   // one DMA thread per CTA: frees the LSU and registers of the other threads
  std::string mapping = "compact";
  std::vector<size_t> sizes;
  bool sweep = false;
  int iters = 10;
  bool fused_triad = false;
  bool verify = true;
  bool cpu = false;  // --cpu: host-only plumbing run (threads as ranks, memcpy as the transport)
  std::string json_path;
  CopyTuning tune;
  uint64_t timeout_ns = 20ull * 1000 * 1000 * 1000;
};

constexpr size_t kReferenceBytes = 1179648ull * 40 * sizeof(float);  // 188 743 680

void usage() {
  std::cout
      << "Usage: peer2pear [label] [options]\n"
         "  label                    free text echoed in the result lines (default Tile2Tile)\n"
         "  -n, --ranks N            ranks = GPUs used, paired (0,1)(2,3)...; default all\n"
         "  --transport put|get|sendrecv|memcpy   default put\n"
         "        put      one-sided: kernel stores into the peer + release flag   (MPI_Put+fence)\n"
         "        get      one-sided: kernel loads from the peer\n"
         "        sendrecv two-sided rendezvous: receiver posts, sender waits+puts (Isend/Irecv)\n"
         "        memcpy   cudaMemcpyPeerAsync copy-engine baseline\n"
         "  --engine tma|ldst        TMA bulk copies through an smem ring (default), or 128-bit ld/st from all threads\n"
         "  --bytes B                message size (default 188743680, the reference size)\n"
         "  --sweep                  1 KiB .. 1 GiB in powers of two plus the reference size\n"
         "  --iters N                timed iterations, minimum reported (default 10)\n"
         "  --mapping compact|spread|compact_plan   rank -> GPU policy (default compact)\n"
         "  --fused-triad            fused a=b+s*c + put of a (one kernel) instead of a plain copy\n"
         "  --no-verify              skip the exact receiver-side check\n"
         "  --ctas N --threads N --unroll N --vec 16|32 --blocked --stages N --stage-kb N   kernel tuning\n"
         "  --json FILE              append one JSON row per size/direction\n"
         "  --cpu                    host-only plumbing run: ranks are threads, the transport is memcpy\n";
}

Config parse(int argc, char** argv) {
  Config c;
  // Program-name personalities of the reference's two builds (p2p/run.sh:4-5): `peer2pear_i` is the two-sided
  // Isend/Irecv build, `peer2pear_w` the one-sided -DUSE_WIN (Put + fence) build.
  {
    std::string self = argc > 0 ? argv[0] : "";
    self = self.substr(self.find_last_of('/') + 1);
    if (self == "peer2pear_i") c.transport = "sendrecv";
    if (self == "peer2pear_w") c.transport = "put";
  }
  bool have_label = false;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto val = [&]() -> std::string {
      if (i + 1 >= argc) HPCP_FAIL("missing value for " + a);
      return argv[++i];
    };
    if (a == "-h" || a == "--help") {
      usage();
      std::exit(0);
    } else if (a == "-n" || a == "--ranks") {
      c.ranks = std::atoi(val().c_str());
    } else if (a == "--transport") {
      c.transport = val();
    } else if (a == "--engine") {
      c.engine = val();
    } else if (a == "--mapping") {
      c.mapping = val();
    } else if (a == "--bytes") {
      c.sizes.push_back(static_cast<size_t>(std::strtoull(val().c_str(), nullptr, 10)));
    } else if (a == "--sweep") {
      c.sweep = true;
    } else if (a == "--iters") {
      c.iters = std::max(1, std::atoi(val().c_str()));
    } else if (a == "--fused-triad") {
      c.fused_triad = true;
    } else if (a == "--no-verify") {
      c.verify = false;
    } else if (a == "--cpu") {
      c.cpu = true;
    } else if (a == "--json") {
      c.json_path = val();
    } else if (a == "--ctas") {
      c.tune.ctas = std::atoi(val().c_str());
    } else if (a == "--threads") {
      c.tune.threads = std::atoi(val().c_str());
    } else if (a == "--unroll") {
      c.tune.unroll = std::atoi(val().c_str());
    } else if (a == "--stages") {
      c.tune.stages = std::atoi(val().c_str());
    } else if (a == "--stage-kb") {
      c.tune.stage_kb = std::atoi(val().c_str());
    } else if (a == "--vec") {
      c.tune.vec_bytes = std::atoi(val().c_str());
    } else if (a == "--blocked") {
      c.tune.blocked = 1;
    } else if (a == "--timeout-s") {
      c.timeout_ns = static_cast<uint64_t>(std::atof(val().c_str()) * 1e9);
    } else if (!a.empty() && a[0] == '-') {
      HPCP_FAIL("unknown option " + a);
    } else if (!have_label) {
      c.label = a;
      have_label = true;
    } else {
      HPCP_FAIL("unexpected argument " + a);
    }
  }
  if (c.sweep) {
    for (size_t b = 1024; b <= (1ull << 30); b <<= 1) c.sizes.push_back(b);
    c.sizes.push_back(kReferenceBytes);
    std::sort(c.sizes.begin(), c.sizes.end());
    c.sizes.erase(std::unique(c.sizes.begin(), c.sizes.end()), c.sizes.end());
  }
  if (c.sizes.empty()) c.sizes.push_back(kReferenceBytes);
  for (size_t b : c.sizes) HPCP_REQUIRE(b >= 16 && b % 16 == 0, "message sizes must be multiples of 16 bytes");
  HPCP_REQUIRE(c.transport == "put" || c.transport == "get" || c.transport == "sendrecv" ||
                   c.transport == "memcpy",
               "unknown transport " + c.transport);
  HPCP_REQUIRE(c.engine == "ldst" || c.engine == "tma", "unknown engine " + c.engine);
  return c;
}

struct Shared {
  const Config* cfg = nullptr;
  NodeMemory* mem = nullptr;
  SymmetricBuffer send, recv, pads, aux;  // aux: triad inputs b|c when --fused-triad
  std::vector<double> uni_ns, bi_ns;      // per size, filled by rank 0
  std::vector<unsigned long long> mismatches;
};

uint32_t* pad_of(const Shared& sh, int r) { return static_cast<uint32_t*>(sh.pads.ptr[r]); }

// One timed phase for one message size.  `sends_to` / `recvs_from` are -1 when idle.
double timed_phase(RankCtx& ctx, Shared& sh, size_t bytes, int sends_to, int recvs_from,
                   cudaStream_t stream, uint32_t& epoch, uint32_t& ticket_issued,
                   uint32_t& barrier_epoch) {
  const Config& cfg = *sh.cfg;
  const int me = ctx.rank;
  const int dev = sh.mem->device(me);
  const CopyEngine engine = cfg.engine == "tma" ? CopyEngine::kTma : CopyEngine::kLdSt;
  uint32_t* my_pad = pad_of(sh, me);
  uint32_t* status = my_pad + kPadWords;
  std::vector<uint32_t*> pad_list;
  for (int r = 0; r < ctx.world; ++r) pad_list.push_back(pad_of(sh, r));

  cudaEvent_t e0, e1;
  HPCP_CUDA(cudaEventCreate(&e0));
  HPCP_CUDA(cudaEventCreate(&e1));
  double best_ns = std::numeric_limits<double>::max();

  NvtxRange phase_range(cfg.transport + (sends_to >= 0 && recvs_from >= 0 ? " bi " : " uni ") +
                        std::to_string(bytes) + " B");
  for (int it = 0; it < cfg.iters; ++it) {
    NvtxRange iter_range("iteration");
    ++epoch;
    ctx.barrier();  // host: everybody has enqueued nothing yet for this iteration
    launch_barrier_all(pad_list.data(), me, ctx.world, ++barrier_epoch, cfg.timeout_ns, status, stream);
    HPCP_CUDA(cudaEventRecord(e0, stream));

    if (cfg.transport == "sendrecv" && recvs_from >= 0)  // post the receive
      launch_signal(pad_of(sh, recvs_from) + kPadReady + me, epoch, stream);

    if (sends_to >= 0 && cfg.transport != "get") {
      SyncOps sync;
      sync.signal_flag = pad_of(sh, sends_to) + kPadDone + me;
      sync.signal_epoch = epoch;
      sync.ticket = my_pad + kPadLocal;
      sync.ticket_base = ticket_issued;
      sync.timeout_ns = cfg.timeout_ns;
      sync.status = status;
      if (cfg.transport == "sendrecv") {
        sync.wait_flag = my_pad + kPadReady + sends_to;
        sync.wait_epoch = epoch;
      }
      if (cfg.transport == "memcpy") {
        HPCP_CUDA(cudaMemcpyPeerAsync(sh.recv.ptr[sends_to], sh.mem->device(sends_to),
                                      sh.send.ptr[me], dev, bytes, stream));
        launch_signal(sync.signal_flag, epoch, stream);
      } else if (cfg.fused_triad) {
        TriadPutArgs t;
        t.a_local = static_cast<float*>(sh.send.ptr[me]);
        t.a_peer = static_cast<float*>(sh.recv.ptr[sends_to]);
        t.b = static_cast<const float*>(sh.aux.ptr[me]);
        t.c = t.b + sh.aux.bytes / sizeof(float) / 2;
        t.s = 3.0f;
        t.n = bytes / sizeof(float);
        ticket_issued += launch_triad_put(t, engine, cfg.tune, sync, nullptr, 0, dev, stream);
      } else {
        ticket_issued += launch_copy(sh.recv.ptr[sends_to], sh.send.ptr[me], bytes,
                                     /*src_is_peer=*/false, engine, cfg.tune, sync, dev, stream);
      }
    }
    if (recvs_from >= 0) {
      if (cfg.transport == "get") {
        SyncOps sync;
        sync.signal_flag = pad_of(sh, recvs_from) + kPadAck + me;  // "your buffer is free again"
        sync.signal_epoch = epoch;
        sync.ticket = my_pad + kPadLocal;
        sync.ticket_base = ticket_issued;
        sync.timeout_ns = cfg.timeout_ns;
        sync.status = status;
        ticket_issued += launch_copy(sh.recv.ptr[me], sh.send.ptr[recvs_from], bytes,
                                     /*src_is_peer=*/true, engine, cfg.tune, sync, dev, stream);
      } else {
        launch_wait(my_pad + kPadDone + recvs_from, epoch, cfg.timeout_ns, status, stream);
      }
    }
    if (cfg.transport == "get" && sends_to >= 0)  // data owner: wait until the reader is done
      launch_wait(my_pad + kPadAck + sends_to, epoch, cfg.timeout_ns, status, stream);

    HPCP_CUDA(cudaEventRecord(e1, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    uint32_t st = 0;
    HPCP_CUDA(cudaMemcpy(&st, status, sizeof st, cudaMemcpyDeviceToHost));
    HPCP_REQUIRE(st == kStatusOk, "rank " + std::to_string(me) +
                                      ": device-side wait timed out (peer did not signal)");
    float ms = 0;
    HPCP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double t_ns = ctx.max(static_cast<double>(ms) * 1e6);  // max over ranks
    best_ns = std::min(best_ns, t_ns);
  }
  (void)cudaEventDestroy(e0);
  (void)cudaEventDestroy(e1);
  return best_ns;
}

unsigned long long verify_recv(Shared& sh, int me, int from, size_t bytes, cudaStream_t stream) {
  const Config& cfg = *sh.cfg;
  unsigned long long* counters = nullptr;
  HPCP_CUDA(cudaMalloc(&counters, 2 * sizeof(unsigned long long)));
  HPCP_CUDA(cudaMemsetAsync(counters, 0, 2 * sizeof(unsigned long long), stream));
  if (cfg.fused_triad)
    launch_verify_triad(static_cast<const float*>(sh.recv.ptr[me]), bytes / sizeof(float), from, 3.0f,
                        counters, stream);
  else
    launch_verify_pattern(static_cast<const uint32_t*>(sh.recv.ptr[me]), bytes / 4,
                          0x9E3779B9u * static_cast<uint32_t>(from + 1), counters, counters + 1,
                          nullptr, 0, 0, nullptr, stream);
  unsigned long long host[2] = {0, 0};
  HPCP_CUDA(cudaMemcpyAsync(host, counters, sizeof host, cudaMemcpyDeviceToHost, stream));
  HPCP_CUDA(cudaStreamSynchronize(stream));
  (void)cudaFree(counters);
  return host[0];
}

void rank_main(RankCtx& ctx, Shared& sh) {
  const Config& cfg = *sh.cfg;
  const int me = ctx.rank;
  const int dev = sh.mem->device(me);
  HPCP_CUDA(cudaSetDevice(dev));
  cudaStream_t stream;
  HPCP_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  const int partner = me ^ 1;
  const bool even = (me % 2) == 0;
  uint32_t epoch = 0, ticket_issued = 0, barrier_epoch = 0;

  for (size_t si = 0; si < cfg.sizes.size(); ++si) {
    const size_t bytes = cfg.sizes[si];
    // Payload: a seeded bijection of the index per sender (exactly checkable).
    if (cfg.fused_triad) {
      float* b = static_cast<float*>(sh.aux.ptr[me]);
      launch_fill_triad_inputs(b, b + sh.aux.bytes / sizeof(float) / 2, bytes / sizeof(float), me, stream);
    } else {
      launch_fill_pattern(static_cast<uint32_t*>(sh.send.ptr[me]), bytes / 4,
                          0x9E3779B9u * static_cast<uint32_t>(me + 1), stream);
    }
    HPCP_CUDA(cudaMemsetAsync(sh.recv.ptr[me], 0, bytes, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    ctx.barrier();

    // Phase 1: unidirectional, even -> odd.
    const double uni = timed_phase(ctx, sh, bytes, even ? partner : -1, even ? -1 : partner, stream,
                                   epoch, ticket_issued, barrier_epoch);
    unsigned long long bad = 0;
    if (cfg.verify && !even) bad += verify_recv(sh, me, partner, bytes, stream);
    HPCP_CUDA(cudaMemsetAsync(sh.recv.ptr[me], 0, bytes, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    ctx.barrier();

    // Phase 2: bidirectional, both directions at once.
    const double bi = timed_phase(ctx, sh, bytes, partner, partner, stream, epoch, ticket_issued,
                                  barrier_epoch);
    if (cfg.verify) bad += verify_recv(sh, me, partner, bytes, stream);
    const double total_bad = ctx.sum(static_cast<double>(bad));
    if (me == 0) {
      sh.uni_ns[si] = uni;
      sh.bi_ns[si] = bi;
      sh.mismatches[si] = static_cast<unsigned long long>(total_bad);
    }
    ctx.barrier();
  }
  (void)cudaStreamDestroy(stream);
}


// ---------------------------------------------------------------- host-only path ----
// Same pairing, phases, iteration/min logic, bandwidth formulas, payload and exact verification, with
// host buffers and memcpy standing in for the NVLink transports: the program logic can be exercised on a
// machine without a GPU.
uint32_t host_pattern_word(size_t i, uint32_t seed) { return pattern_word(i, seed); }

int run_on_host(const Config& cfg) {
  const int P = cfg.ranks > 0 ? cfg.ranks : 2;
  HPCP_REQUIRE(P >= 2 && P % 2 == 0, "peer2pear: need an even number of ranks >= 2");
  const int pairs = P / 2;
  int rc = 0;
  for (size_t bytes : cfg.sizes) {
    const size_t words = bytes / 4;
    std::vector<std::vector<uint32_t>> send(P, std::vector<uint32_t>(words)), recv(P, std::vector<uint32_t>(words));
    double uni_ns = 0, bi_ns = 0;
    unsigned long long mismatches = 0;
    run_ranks(P, [&](RankCtx& ctx) {
      const int me = ctx.rank, partner = me ^ 1;
      const bool even = me % 2 == 0;
      const uint32_t seed = 0x9E3779B9u * static_cast<uint32_t>(me + 1);
      for (size_t i = 0; i < words; ++i) send[me][i] = host_pattern_word(i, seed);
      auto phase = [&](bool sends, bool receives) {
        double best = std::numeric_limits<double>::max();
        for (int it = 0; it < cfg.iters; ++it) {
          ctx.barrier();
          const auto t0 = std::chrono::steady_clock::now();
          if (sends) std::memcpy(recv[partner].data(), send[me].data(), bytes);  // "put" into the partner
          ctx.barrier();                                                         // fence: all puts landed
          (void)receives;
          const double ns = std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t0).count();
          best = std::min(best, ctx.max(ns));
        }
        return best;
      };
      auto check = [&](int from) {
        const uint32_t s = 0x9E3779B9u * static_cast<uint32_t>(from + 1);
        unsigned long long bad = 0;
        for (size_t i = 0; i < words; ++i) bad += recv[me][i] != host_pattern_word(i, s);
        return bad;
      };
      const double uni = phase(even, !even);
      unsigned long long bad = (cfg.verify && !even) ? check(partner) : 0;
      std::fill(recv[me].begin(), recv[me].end(), 0u);
      const double bi = phase(true, true);
      if (cfg.verify) bad += check(partner);
      const double all_bad = ctx.sum(static_cast<double>(bad));
      if (me == 0) {
        uni_ns = uni;
        bi_ns = bi;
        mismatches = static_cast<unsigned long long>(all_bad);
      }
    });
    std::string label = cfg.label;
    if (cfg.sizes.size() > 1) label += " [" + std::to_string(bytes) + " B]";
    std::cout << label << " Unidirectional Bandwidth: " << static_cast<double>(bytes) * pairs / uni_ns << " GB/s"
              << std::endl;
    std::cout << label << " Bidirectional Bandwidth: " << 2.0 * static_cast<double>(bytes) * pairs / bi_ns << " GB/s"
              << std::endl;
    if (mismatches != 0) {
      std::cout << label << " VERIFICATION FAILED: " << mismatches << " wrong words" << std::endl;
      rc = 1;
    }
    if (!cfg.json_path.empty()) {  // same row shape as the GPU path; engine "host" marks the plumbing run
      std::ofstream f(cfg.json_path, std::ios::app);
      const double uni_bw = static_cast<double>(bytes) * pairs / uni_ns;
      f << "{\"pattern\":\"peer2pear\",\"label\":\"" << cfg.label << "\",\"transport\":\"" << cfg.transport
        << "\",\"engine\":\"host\",\"fused_triad\":false,\"mapping\":\"" << cfg.mapping << "\",\"ranks\":" << P
        << ",\"bytes\":" << bytes << ",\"uni_us\":" << uni_ns * 1e-3 << ",\"bi_us\":" << bi_ns * 1e-3
        << ",\"uni_GBps\":" << uni_bw << ",\"bi_GBps\":" << 2.0 * static_cast<double>(bytes) * pairs / bi_ns
        << ",\"uni_GBps_per_pair\":" << uni_bw / pairs << ",\"frac_of_450GBps_per_dir\":" << (uni_bw / pairs) / 450.0
        << ",\"mismatches\":" << mismatches << "}\n";
    }
  }
  return rc;
}
}  // namespace

int main(int argc, char** argv) {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  try {
    Config cfg = parse(argc, argv);
    if (cfg.cpu) return run_on_host(cfg);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
      std::cerr << "peer2pear: no CUDA device visible" << std::endl;
      return 1;
    }
    if (cfg.ranks <= 0) cfg.ranks = ndev - (ndev % 2);
    if (cfg.ranks < 2 || cfg.ranks % 2 != 0) {
      std::cerr << "peer2pear: need an even number of ranks >= 2 (have " << ndev << " GPU(s))"
                << std::endl;
      return 1;
    }

    // rank -> device (in-process equivalent of tile_mapping.sh).
    std::vector<std::vector<int>> planes;
    if (cfg.mapping == "compact_plan") {
      topo::Fabric fabric;
      std::string why;
      if (topo::fabric_from_nvml(&fabric, &why))
        planes = topo::merge_planes(static_cast<int>(fabric.gpus.size()), fabric.links);
      else
        std::cerr << "# compact_plan: " << why << "; falling back to ordinal order" << std::endl;
    }
    std::vector<int> devices;
    for (int r = 0; r < cfg.ranks; ++r)
      devices.push_back(topo::device_for_rank(cfg.mapping, r, ndev, planes) % ndev);

    // Ranks that share a GPU (more ranks than devices) must leave each other room: a copy kernel that waits in its
    // prologue for the peer's "receive posted" word holds its SM slots while the peer's signal kernel needs one on the
    // SAME GPU.  Half a wave of CTAs per sharing rank keeps registers and thread slots free.
    int ranks_per_dev = 1;
    for (int d = 0; d < ndev; ++d)
      ranks_per_dev = std::max<int>(ranks_per_dev, static_cast<int>(std::count(devices.begin(), devices.end(), d)));
    if (ranks_per_dev > 1 && cfg.tune.ctas == 0)
      cfg.tune.ctas = std::max(1, device_sm_count(devices[0]) / ranks_per_dev);

    NodeMemory mem(devices);
    Shared sh;
    sh.cfg = &cfg;
    sh.mem = &mem;
    const size_t max_bytes = *std::max_element(cfg.sizes.begin(), cfg.sizes.end());
    sh.send = mem.alloc(max_bytes);
    sh.recv = mem.alloc(max_bytes);
    sh.pads = mem.alloc_pads();
    if (cfg.fused_triad) sh.aux = mem.alloc(2 * max_bytes);
    sh.uni_ns.assign(cfg.sizes.size(), 0);
    sh.bi_ns.assign(cfg.sizes.size(), 0);
    sh.mismatches.assign(cfg.sizes.size(), 0);

    run_ranks(cfg.ranks, [&](RankCtx& ctx) { rank_main(ctx, sh); });

    const int pairs = cfg.ranks / 2;
    int rc = 0;
    for (size_t si = 0; si < cfg.sizes.size(); ++si) {
      const double bytes = static_cast<double>(cfg.sizes[si]);
      const double uni_bw = bytes * pairs / sh.uni_ns[si];        // bytes/ns == GB/s
      const double bi_bw = 2.0 * bytes * pairs / sh.bi_ns[si];
      std::string label = cfg.label;
      if (cfg.sizes.size() > 1) label += " [" + std::to_string(cfg.sizes[si]) + " B]";
      std::cout << label << " Unidirectional Bandwidth: " << uni_bw << " GB/s" << std::endl;
      std::cout << label << " Bidirectional Bandwidth: " << bi_bw << " GB/s" << std::endl;
      if (cfg.verify && sh.mismatches[si] != 0) {
        std::cout << label << " VERIFICATION FAILED: " << sh.mismatches[si] << " wrong words"
                  << std::endl;
        rc = 1;
      }
      if (!cfg.json_path.empty()) {
        std::ofstream f(cfg.json_path, std::ios::app);
        f << "{\"pattern\":\"peer2pear\",\"label\":\"" << cfg.label << "\",\"transport\":\""
          << cfg.transport << "\",\"engine\":\"" << cfg.engine << "\",\"fused_triad\":"
          << (cfg.fused_triad ? "true" : "false") << ",\"mapping\":\"" << cfg.mapping
          << "\",\"ranks\":" << cfg.ranks << ",\"bytes\":" << cfg.sizes[si]
          << ",\"uni_us\":" << sh.uni_ns[si] * 1e-3 << ",\"bi_us\":" << sh.bi_ns[si] * 1e-3
          << ",\"uni_GBps\":" << uni_bw << ",\"bi_GBps\":" << bi_bw
          << ",\"uni_GBps_per_pair\":" << uni_bw / pairs
          << ",\"frac_of_450GBps_per_dir\":" << (uni_bw / pairs) / 450.0
          << ",\"mismatches\":" << sh.mismatches[si] << "}\n";
      }
    }
    mem.free(sh.send);
    mem.free(sh.recv);
    mem.free(sh.pads);
    if (cfg.fused_triad) mem.free(sh.aux);
    return rc;
  } catch (const std::exception& e) {
    std::cerr << "peer2pear: ERROR: " << e.what() << std::endl;
    return 1;
  }
}
