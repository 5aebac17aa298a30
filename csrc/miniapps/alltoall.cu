// alltoall — the equal-block all-to-all (↔ MPI_Alltoall, ncclAllToAll) in one launch per rank.
//
//   alltoall [-n ranks] [--block-bytes B] [--pull] [--stock memcpy] [--sweep] [--iters N] [--warmup N] [--ctas N]
//            [--json FILE] [--cpu]
//
// Every rank holds a send and a receive buffer of P blocks of B bytes (default 16 MiB: 128 MiB of send buffer per rank
// at P = 8).  Afterwards block p of rank r's receive buffer is block r of rank p's send buffer.  The kernel (push by
// default, --pull for peer loads) is csrc/kernels/all_to_all.cu.  --stock memcpy is the stock shape as a measured
// baseline: P cudaMemcpyAsync peer copies per rank, then a cross-rank barrier.  --sweep runs B = 16 B ... 256 MiB in
// powers of two (with --block-bytes: up to that size), one report line and one JSON row each.  --cpu is the host-only
// plumbing run: ranks are threads, the same staggered walk is memcpy + a barrier.
//
// Check (outside the timed region, before every iteration): block q of rank r's send buffer gets the seeded pattern of
// the ordered pair (r, q) and of the iteration, the receive buffer a poison seed no pair uses.  After the last
// iteration every receive block p of rank r is checked word for word against the seed of (p, r): a block sent to the
// wrong rank or slot, a block never sent (the local one included), a short tail and a result of an earlier iteration
// each leave wrong words.  Ranks are placed on GPUs as devices.hpp does.
#include <getopt.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <limits>
#include <string>
#include <vector>

#include "../common/cuda_check.h"
#include "../common/nvtx.h"
#include "../common/peer_mem.h"
#include "../common/rank_runtime.h"
#include "../common/signal_layout.h"
#include "../kernels/api.h"
#include "../kernels/payload.h"
#include "devices.hpp"

namespace {

using namespace hpcp;

struct Config {
  int ranks = -1;  // -1: every GPU (--cpu: 4)
  size_t block_bytes = size_t{16} << 20;
  bool block_given = false;
  bool pull = false;
  std::string stock;  // "" or "memcpy"
  bool sweep = false;
  int iters = 5;
  int warmup = 1;
  int ctas = 0;
  uint64_t timeout_ns = 30ull * 1000 * 1000 * 1000;
  std::string json_path;
  bool cpu = false;
};

constexpr size_t kSweepMaxBytes = size_t{256} << 20;

void print_help() {
  std::cout << "Usage: alltoall [options]\n"
               "options:\n"
               " -n N               ranks (one host thread + one GPU each; default: all GPUs; more ranks than GPUs are\n"
               "                    placed round-robin); 1 ... 16\n"
               " --block-bytes B    bytes per block, a positive multiple of 16 (default 16 MiB); with --sweep the largest\n"
               " --pull             the kernel loads from the peers' send buffers instead of storing into their receive\n"
               "                    buffers\n"
               " --stock memcpy     stock shape: P cudaMemcpyAsync peer copies per rank, then a cross-rank barrier\n"
               " --sweep            block sizes 16 B ... 256 MiB (or --block-bytes) in powers of two\n"
               " --iters N --warmup N  timed / untimed repetitions (min is reported)\n"
               " --ctas N           CTAs per rank\n"
               " --json FILE        append one JSON row per block size\n"
               " --cpu              host-only plumbing run: ranks are threads, the walk is memcpy + a barrier\n";
}

// The pattern seed of block `dst` of rank `src`'s send buffer in iteration `it`: unique per ordered pair and iteration
// (bit 30 set, bit 31 clear), so no seed is ever the poison.
uint32_t pair_seed(uint32_t it, int src, int dst) {
  return 0x40000000u | ((it & 0x3fffffu) << 8) | (static_cast<uint32_t>(src) << 4) | static_cast<uint32_t>(dst);
}
constexpr uint32_t kPoisonSeed = 0xC0DE0000u;

const char* variant_name(const Config& cfg) {
  return cfg.cpu ? "host" : cfg.stock == "memcpy" ? "memcpy" : cfg.pull ? "pull" : "push";
}

std::vector<size_t> block_sizes(const Config& cfg) {
  if (!cfg.sweep) return {cfg.block_bytes};
  const size_t top = cfg.block_given ? cfg.block_bytes : kSweepMaxBytes;
  std::vector<size_t> out;
  for (size_t b = 16; b <= top; b *= 2) out.push_back(b);
  return out;
}

struct Row {
  size_t block_bytes = 0;
  double ms = 0;
  unsigned long long bad = 0;
  int ctas = 0;
};

// GB/s sent per rank: (P-1) blocks cross a link, the local one does not.
void report(const Config& cfg, int P, const Row& r) {
  const double sent = static_cast<double>(P - 1) * static_cast<double>(r.block_bytes);
  const double gbps = r.ms > 0 ? sent / (r.ms * 1e-3) * 1e-9 : 0.0;
  const char* algo = cfg.cpu ? "host-alltoall" : variant_name(cfg);
  std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << r.ms << " ms | alltoall " << algo
            << " P=" << P << " B=" << r.block_bytes << (cfg.cpu ? " host-threads" : "") << " | " << gbps
            << " GB/s sent per rank" << std::endl;
  if (!cfg.json_path.empty()) {
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      std::fprintf(f,
                   "{\"pattern\":\"alltoall\",\"variant\":\"%s\",\"ranks\":%d,\"block_bytes\":%zu,\"ms\":%.6f,"
                   "\"GBps_sent_per_rank\":%.3f,\"ctas\":%d,\"mismatches\":%llu}\n",
                   variant_name(cfg), P, r.block_bytes, r.ms, gbps, r.ctas, r.bad);
      std::fclose(f);
    }
  }
}

// One write per line: the ranks are threads that print at the same time.
void print_verdict(int me, unsigned long long bad) {
  const std::string line = bad == 0 ? "Passed " + std::to_string(me) + "\n"
                                    : "FAILED " + std::to_string(me) + ": " + std::to_string(bad) + " wrong words\n";
  std::cout << line << std::flush;
}

// ------------------------------------------------------------------------------------------------------- GPU ----
struct Shared {
  Config cfg;
  NodeMemory* mem = nullptr;
  SymmetricBuffer send, recv, pads;
  std::vector<Row> rows;  // written by rank 0
};

void rank_main(RankCtx& ctx, Shared& sh) {
  const Config& cfg = sh.cfg;
  const int me = ctx.rank, P = ctx.world;
  const int dev = sh.mem->device(me);
  HPCP_CUDA(cudaSetDevice(dev));
  cudaStream_t stream;
  HPCP_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  std::vector<uint32_t*> pads;
  for (int r = 0; r < P; ++r) pads.push_back(static_cast<uint32_t*>(sh.pads.ptr[r]));
  uint32_t* my_pad = pads[me];
  uint32_t* status = my_pad + kPadWords;
  unsigned char* my_send = static_cast<unsigned char*>(sh.send.ptr[me]);
  unsigned char* my_recv = static_cast<unsigned char*>(sh.recv.ptr[me]);
  unsigned long long* count = nullptr;
  HPCP_CUDA(cudaMalloc(&count, sizeof *count));
  cudaEvent_t e0, e1;
  HPCP_CUDA(cudaEventCreate(&e0));
  HPCP_CUDA(cudaEventCreate(&e1));
  uint32_t barrier_epoch = 0, ticket_issued = 0, it_global = 0;

  for (const size_t B : block_sizes(cfg)) {
    double best_ms = std::numeric_limits<double>::max();
    int ctas = 0;
    for (int it = 0; it < cfg.warmup + cfg.iters; ++it, ++it_global) {
      NvtxRange range(it < cfg.warmup ? "alltoall warm-up" : "alltoall timed");
      for (int q = 0; q < P; ++q)
        launch_fill_pattern(reinterpret_cast<uint32_t*>(my_send + q * B), B / 4, pair_seed(it_global, me, q), stream);
      launch_fill_pattern(reinterpret_cast<uint32_t*>(my_recv), P * B / 4, kPoisonSeed, stream);
      HPCP_CUDA(cudaStreamSynchronize(stream));
      ctx.barrier();
      launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
      HPCP_CUDA(cudaEventRecord(e0, stream));
      if (cfg.stock == "memcpy") {
        for (int j = 0; j < P; ++j) {
          const int p = (me + 1 + j) % P;
          HPCP_CUDA(cudaMemcpyAsync(static_cast<unsigned char*>(sh.recv.ptr[p]) + me * B, my_send + p * B, B,
                                    cudaMemcpyDefault, stream));
        }
        launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
      } else {
        AllToAllArgs a;
        for (int r = 0; r < P; ++r) {
          a.send[r] = sh.send.ptr[r];
          a.recv[r] = sh.recv.ptr[r];
          a.pads[r] = pads[r];
        }
        a.ticket = my_pad + kPadLocal;
        a.ticket_base = ticket_issued;
        a.rank = me;
        a.world = P;
        a.block_bytes = B;
        a.barrier_epoch = ++barrier_epoch;
        a.timeout_ns = cfg.timeout_ns;
        a.status = status;
        a.pull = cfg.pull;
        ctas = launch_all_to_all(a, cfg.ctas, dev, stream);
        ticket_issued += static_cast<uint32_t>(ctas);
      }
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
    // Every receive block p against the seed of (p, me) in the last iteration.
    HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
    for (int p = 0; p < P; ++p)
      launch_verify_pattern(reinterpret_cast<const uint32_t*>(my_recv + p * B), B / 4, pair_seed(it_global - 1, p, me),
                            count, nullptr, nullptr, 0, 0, nullptr, stream);
    unsigned long long bad = 0;
    HPCP_CUDA(cudaMemcpyAsync(&bad, count, sizeof bad, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    const double total_bad = ctx.sum(static_cast<double>(bad));
    print_verdict(me, bad);
    if (me == 0) sh.rows.push_back({B, best_ms, static_cast<unsigned long long>(total_bad), ctas});
    ctx.barrier();
    if (me == 0) report(cfg, P, sh.rows.back());
    ctx.barrier();
  }
  (void)cudaFree(count);
  (void)cudaEventDestroy(e0);
  (void)cudaEventDestroy(e1);
  (void)cudaStreamDestroy(stream);
}

// ---------------------------------------------------------------------------------------------- host-only path ----
// Ranks are threads of the rank runtime; the kernel's staggered walk (block j goes to peer (rank + 1 + j) % P, the
// local block last) is a memcpy per block, then a barrier.  No GPU: the plumbing configuration that tests options,
// walk, check and output on a machine without a device.
int run_on_host(const Config& cfg) {
  const int P = cfg.ranks;
  const std::vector<size_t> sizes = block_sizes(cfg);
  const size_t top = *std::max_element(sizes.begin(), sizes.end());
  std::vector<std::vector<uint32_t>> send(P), recv(P);
  std::vector<Row> rows;
  run_ranks(P, [&](RankCtx& ctx) {
    const int me = ctx.rank;
    send[me].resize(P * top / 4);
    recv[me].resize(P * top / 4);
    uint32_t it_global = 0;
    for (const size_t B : sizes) {
      const size_t words = B / 4;
      double best_ms = std::numeric_limits<double>::max();
      for (int it = 0; it < cfg.warmup + cfg.iters; ++it, ++it_global) {
        for (int q = 0; q < P; ++q)
          for (size_t i = 0; i < words; ++i) send[me][q * words + i] = pattern_word(i, pair_seed(it_global, me, q));
        for (size_t i = 0; i < P * words; ++i) recv[me][i] = pattern_word(i, kPoisonSeed);
        ctx.barrier();
        const auto t0 = std::chrono::steady_clock::now();
        for (int j = 0; j < P; ++j) {
          const int p = (me + 1 + j) % P;
          std::memcpy(recv[p].data() + me * words, send[me].data() + p * words, B);
        }
        ctx.barrier();
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        const double t = ctx.max(ms);
        if (it >= cfg.warmup) best_ms = std::min(best_ms, t);
      }
      unsigned long long bad = 0;
      for (int p = 0; p < P; ++p) {
        const uint32_t seed = pair_seed(it_global - 1, p, me);
        for (size_t i = 0; i < words; ++i) bad += recv[me][p * words + i] != pattern_word(i, seed);
      }
      const double total_bad = ctx.sum(static_cast<double>(bad));
      print_verdict(me, bad);
      if (me == 0) rows.push_back({B, best_ms, static_cast<unsigned long long>(total_bad), 0});
      ctx.barrier();
      if (me == 0) report(cfg, P, rows.back());
      ctx.barrier();
    }
  });
  for (const Row& r : rows)
    if (r.bad != 0) return 1;
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  hpcp::prefer_eager_module_loading();  // spin-waiting kernels + lazy module loading can deadlock (cuda_check.h)
  try {
    Shared sh;
    Config& cfg = sh.cfg;
    static const option long_opts[] = {{"block-bytes", required_argument, nullptr, 1},
                                       {"pull", no_argument, nullptr, 2},
                                       {"stock", required_argument, nullptr, 3},
                                       {"sweep", no_argument, nullptr, 4},
                                       {"iters", required_argument, nullptr, 5},
                                       {"warmup", required_argument, nullptr, 6},
                                       {"ctas", required_argument, nullptr, 7},
                                       {"json", required_argument, nullptr, 8},
                                       {"cpu", no_argument, nullptr, 9},
                                       {"help", no_argument, nullptr, 'h'},
                                       {nullptr, 0, nullptr, 0}};
    int opt;
    while ((opt = getopt_long(argc, argv, "hn:", long_opts, nullptr)) != -1) {
      switch (opt) {
        case 'h': print_help(); return 0;
        case 'n': cfg.ranks = std::atoi(optarg); break;
        case 1: {
          char* end = nullptr;
          cfg.block_bytes = std::strtoull(optarg, &end, 10);
          HPCP_REQUIRE(end != optarg && *end == '\0' && optarg[0] != '-', std::string("--block-bytes: not a byte count: ") + optarg);
          cfg.block_given = true;
          break;
        }
        case 2: cfg.pull = true; break;
        case 3: cfg.stock = optarg; break;
        case 4: cfg.sweep = true; break;
        case 5: cfg.iters = std::max(1, std::atoi(optarg)); break;
        case 6: cfg.warmup = std::max(0, std::atoi(optarg)); break;
        case 7: cfg.ctas = std::atoi(optarg); break;
        case 8: cfg.json_path = optarg; break;
        case 9: cfg.cpu = true; break;
        default: print_help(); return 1;
      }
    }
    // Usage errors, before anything is allocated.
    HPCP_REQUIRE(cfg.stock.empty() || cfg.stock == "memcpy", "--stock must be memcpy, not " + cfg.stock);
    HPCP_REQUIRE(cfg.stock.empty() || !cfg.pull, "--stock memcpy is refused with --pull: the stock shape has no pull");
    HPCP_REQUIRE(cfg.stock.empty() || !cfg.cpu, "--stock memcpy is a GPU baseline: --cpu runs the host walk only");
    if (cfg.cpu && cfg.ranks < 0) cfg.ranks = 4;
    if (const char* why = all_to_all_refusal(cfg.ranks < 0 ? 1 : cfg.ranks, cfg.block_bytes)) HPCP_FAIL(why);

    if (cfg.cpu) return run_on_host(cfg);
    const int ndev = visible_device_count();
    if (ndev == 0) {
      std::cerr << "Error: No devices" << std::endl;
      return 1;
    }
    if (cfg.ranks < 0) cfg.ranks = std::min(ndev, kApiMaxRanks);
    const int P = cfg.ranks;
    std::vector<int> devices;
    for (int r = 0; r < P; ++r) devices.push_back(primary_device(r, P, ndev));
    const int ranks_per_dev = (P + ndev - 1) / ndev;
    if (ranks_per_dev > 1 && cfg.ctas == 0)  // every rank's barrier CTA must find a slot next to its peers' grids
      cfg.ctas = std::max(1, device_sm_count(devices[0]) / ranks_per_dev);

    NodeMemory mem(devices);
    sh.mem = &mem;
    const std::vector<size_t> sizes = block_sizes(cfg);
    const size_t bytes = *std::max_element(sizes.begin(), sizes.end()) * P;
    sh.pads = mem.alloc_pads(0);
    sh.send = mem.alloc(bytes, AllocKind::kDevice, /*zero=*/false);
    sh.recv = mem.alloc(bytes, AllocKind::kDevice, /*zero=*/false);
    run_ranks(P, [&](RankCtx& ctx) { rank_main(ctx, sh); });
    mem.free(sh.send);
    mem.free(sh.recv);
    mem.free(sh.pads);
    for (const Row& r : sh.rows)
      if (r.bad != 0) return 1;
    return 0;
  } catch (const std::exception& e) {
    std::cerr << "Error: " << e.what() << std::endl;
    return 1;
  }
}
