// alltoall — the equal-block all-to-all (↔ MPI_Alltoall, ncclAllToAll) in one launch per rank.
//
//   alltoall [-n ranks] [--block-bytes B] [--pull] [--stock memcpy] [--sweep] [--iters N] [--warmup N] [--ctas N]
//            [--json FILE] [--cpu] [--counts random|skewed|equal [--row-bytes R]]
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
//
// --counts runs the all-to-all-v instead (↔ MPI_Alltoallv with packed displacements): rows of R bytes (default 16),
// --block-bytes the mean segment, rounded to rows.  Every iteration draws a new count matrix from a seed: `random`
// gives every ordered pair 0 ... 2*mean rows and one pair none; `skewed` sends 2*mean rows from every rank into one hot
// receiver (rank it % P, exactly at the receive capacity) and at most mean/P into the others; `equal` gives every pair
// the mean (the equal-block exchange through the v kernel, for comparing the two).  Both capacities are
// 2*P*mean rows.  The counts reach the device counts buffers outside the timed region; the kernel reads them there
// and the host never tells it a count.  Check: the segments and the poison as above at their packed rows, recv_counts
// against the host's matrix (not for --stock memcpy, whose copies are placed by the host), and the rows past each
// rank's total still the poison.
//
// Run as `allgather` (a program-name link to this binary) it is the all-gather instead (↔ MPI_Allgather,
// ncclAllGather): every rank holds ONE send block of B bytes and afterwards block p of every rank's receive buffer (P
// blocks) is rank p's.  --pull, --stock memcpy (P-1 peer cudaMemcpyAsync copies plus the local one in the staggered
// order, then the barrier), --sweep, --cpu and --json as above; --counts and --row-bytes are usage errors.  Check: rank
// p's block holds the seed of (p, iteration), the receive buffer the poison; after the last iteration every receive
// block p is checked against the seed of p, and the send block against its own seed (it is never written).
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
#include "../kernels/alltoallv_plan.h"
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
  std::string counts;  // "" (the equal-block kernel), "random", "skewed" or "equal"
  size_t row_bytes = 16;
  bool row_given = false;
  bool gather = false;  // program name `allgather`: the all-gather
};

constexpr size_t kSweepMaxBytes = size_t{256} << 20;

void print_help(bool gather) {
  if (gather) {
    std::cout << "Usage: allgather [options]\n"
                 "options:\n"
                 " -n N               ranks (one host thread + one GPU each; default: all GPUs); 1 ... 16\n"
                 " --block-bytes B    bytes of every rank's send block, a positive multiple of 16 (default 16 MiB);\n"
                 "                    with --sweep the largest\n"
                 " --pull             the kernel loads the peers' blocks instead of storing mine into their buffers\n"
                 " --stock memcpy     stock shape: P cudaMemcpyAsync peer copies per rank, then a cross-rank barrier\n"
                 " --sweep            block sizes 16 B ... 256 MiB (or --block-bytes) in powers of two\n"
                 " --iters N --warmup N  timed / untimed repetitions (min is reported)\n"
                 " --ctas N           CTAs per rank\n"
                 " --json FILE        append one JSON row per block size\n"
                 " --cpu              host-only plumbing run: ranks are threads, the walk is memcpy + a barrier\n";
    return;
  }
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
               " --cpu              host-only plumbing run: ranks are threads, the walk is memcpy + a barrier\n"
               " --counts K         all-to-all-v with device-resident counts drawn per iteration: random | skewed |\n"
               "                    equal (every pair the mean);\n"
               "                    --block-bytes is then the mean segment\n"
               " --row-bytes R      with --counts: bytes per row, a positive multiple of 16 (default 16)\n";
}

// The pattern seed of block `dst` of rank `src`'s send buffer in iteration `it`: unique per ordered pair and iteration
// (bit 30 set, bit 31 clear), so no seed is ever the poison.
uint32_t pair_seed(uint32_t it, int src, int dst) {
  return 0x40000000u | ((it & 0x3fffffu) << 8) | (static_cast<uint32_t>(src) << 4) | static_cast<uint32_t>(dst);
}
constexpr uint32_t kPoisonSeed = 0xC0DE0000u;
// The all-gather's seed of rank `src`'s block in iteration `it` (bit 29 set, bits 30 and 31 clear: never the poison).
uint32_t gather_seed(uint32_t it, int src) { return 0x20000000u | ((it & 0x3fffffu) << 4) | static_cast<uint32_t>(src); }
constexpr uint32_t kTailPoisonSeed = 0xC0DE0001u;  // --counts: the receive rows past the total, never written

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
  double off_rank_bytes = 0;       // --counts: bytes that crossed to another rank in the timed iteration, all ranks
  double max_bytes_into_a_rank = 0;
};

// ------------------------------------------------------------------------------------------- all-to-all-v plan ----
uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Rows of the mean segment: --block-bytes rounded to rows, at least one.
int64_t mean_rows(size_t block_bytes, size_t row_bytes) {
  return std::max<int64_t>(1, static_cast<int64_t>((block_bytes + row_bytes / 2) / row_bytes));
}
int64_t capacity_rows(int P, int64_t mean) { return 2 * static_cast<int64_t>(P) * mean; }

// The count matrix of iteration `it` (row-major, M[p][q] rows from p to q); every one fits the capacities above.
std::vector<int64_t> draw_counts(const std::string& kind, int P, int64_t mean, uint32_t it) {
  std::vector<int64_t> m(static_cast<size_t>(P) * P);
  const int hot = static_cast<int>(it % static_cast<uint32_t>(P));
  for (int p = 0; p < P; ++p)
    for (int q = 0; q < P; ++q) {
      const uint64_t h = mix64((static_cast<uint64_t>(it) << 16) | (static_cast<uint64_t>(p) << 8) | q);
      m[p * P + q] = kind == "equal"    ? mean
                     : kind == "skewed" ? (q == hot ? 2 * mean : static_cast<int64_t>(h % (mean / P + 1)))
                                        : static_cast<int64_t>(h % (2 * mean + 1));
    }
  if (kind == "random") m[mix64(0xA11u ^ (static_cast<uint64_t>(it) << 32)) % m.size()] = 0;
  return m;
}

// Off-rank bytes of all ranks and the most bytes any rank receives.
void count_traffic(const std::vector<int64_t>& m, int P, size_t row_bytes, Row& row) {
  row.off_rank_bytes = row.max_bytes_into_a_rank = 0;
  for (int q = 0; q < P; ++q) {
    double into = 0;
    for (int p = 0; p < P; ++p) {
      const double b = static_cast<double>(m[p * P + q]) * static_cast<double>(row_bytes);
      into += b;
      if (p != q) row.off_rank_bytes += b;
    }
    row.max_bytes_into_a_rank = std::max(row.max_bytes_into_a_rank, into);
  }
}

// GB/s sent per rank: (P-1) blocks cross a link, the local one does not.
void report(const Config& cfg, int P, const Row& r) {
  const double sent = static_cast<double>(P - 1) * static_cast<double>(r.block_bytes);
  const double gbps = r.ms > 0 ? sent / (r.ms * 1e-3) * 1e-9 : 0.0;
  const char* pattern = cfg.gather ? "allgather" : "alltoall";
  const std::string algo = cfg.cpu ? std::string("host-") + pattern : variant_name(cfg);
  std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << r.ms << " ms | " << pattern << " " << algo
            << " P=" << P << " B=" << r.block_bytes << (cfg.cpu ? " host-threads" : "") << " | " << gbps
            << " GB/s sent per rank" << std::endl;
  if (!cfg.json_path.empty()) {
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      std::fprintf(f,
                   "{\"pattern\":\"%s\",\"variant\":\"%s\",\"ranks\":%d,\"block_bytes\":%zu,\"ms\":%.6f,"
                   "\"GBps_sent_per_rank\":%.3f,\"ctas\":%d,\"mismatches\":%llu}\n",
                   pattern, variant_name(cfg), P, r.block_bytes, r.ms, gbps, r.ctas, r.bad);
      std::fclose(f);
    }
  }
}

// GB/s: off-rank bytes summed over ranks, divided by P and by the time (for equal blocks (P-1)*B/t as above).
void report_v(const Config& cfg, int P, const Row& r) {
  const double gbps = r.ms > 0 ? r.off_rank_bytes / P / (r.ms * 1e-3) * 1e-9 : 0.0;
  const char* algo = cfg.cpu ? "host-alltoallv" : variant_name(cfg);
  std::cout << "Elapsed (max over ranks, min of " << cfg.iters << "): " << r.ms << " ms | alltoallv " << algo
            << " " << cfg.counts << " P=" << P << " B=" << r.block_bytes << " R=" << cfg.row_bytes
            << (cfg.cpu ? " host-threads" : "") << " | " << gbps << " GB/s sent per rank" << std::endl;
  if (!cfg.json_path.empty()) {
    if (FILE* f = std::fopen(cfg.json_path.c_str(), "a")) {
      std::fprintf(f,
                   "{\"pattern\":\"alltoallv\",\"variant\":\"%s\",\"ranks\":%d,\"block_bytes\":%zu,\"ms\":%.6f,"
                   "\"GBps_sent_per_rank\":%.3f,\"ctas\":%d,\"mismatches\":%llu,\"counts\":\"%s\",\"row_bytes\":%zu,"
                   "\"max_bytes_into_a_rank\":%.0f}\n",
                   variant_name(cfg), P, r.block_bytes, r.ms, gbps, r.ctas, r.bad, cfg.counts.c_str(), cfg.row_bytes,
                   r.max_bytes_into_a_rank);
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
  SymmetricBuffer send, recv, pads, counts;
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
      if (cfg.gather)
        launch_fill_pattern(reinterpret_cast<uint32_t*>(my_send), B / 4, gather_seed(it_global, me), stream);
      else
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
          HPCP_CUDA(cudaMemcpyAsync(static_cast<unsigned char*>(sh.recv.ptr[p]) + me * B, my_send + (cfg.gather ? 0 : p * B),
                                    B, cudaMemcpyDefault, stream));
        }
        launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
      } else if (cfg.gather) {
        AllGatherArgs a;
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
        ctas = launch_all_gather(a, cfg.ctas, dev, stream);
        ticket_issued += static_cast<uint32_t>(ctas);
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
    // Every receive block p against the seed of (p, me) in the last iteration (all-gather: of p, and my send block
    // against my own seed).
    HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
    for (int p = 0; p < P; ++p)
      launch_verify_pattern(reinterpret_cast<const uint32_t*>(my_recv + p * B), B / 4,
                            cfg.gather ? gather_seed(it_global - 1, p) : pair_seed(it_global - 1, p, me), count, nullptr,
                            nullptr, 0, 0, nullptr, stream);
    if (cfg.gather)
      launch_verify_pattern(reinterpret_cast<const uint32_t*>(my_send), B / 4, gather_seed(it_global - 1, me), count,
                            nullptr, nullptr, 0, 0, nullptr, stream);
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

// Rows every rank sends to rank r under the matrix m.
int64_t rows_into(const std::vector<int64_t>& m, int P, int r) {
  int64_t n = 0;
  for (int p = 0; p < P; ++p) n += m[p * P + r];
  return n;
}

// --counts on the GPU: the counts of iteration it go to this rank's counts buffer, its send segments get their seeds at
// their packed rows, the receive rows get the poison; then the all-to-all-v kernel (or the stock memcpy shape).
void rank_main_v(RankCtx& ctx, Shared& sh) {
  const Config& cfg = sh.cfg;
  const int me = ctx.rank, P = ctx.world;
  const size_t rb = cfg.row_bytes;
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
  int64_t* my_counts = static_cast<int64_t*>(sh.counts.ptr[me]);
  int64_t* recv_counts = nullptr;
  uint32_t* verdict = nullptr;
  unsigned long long* count = nullptr;
  HPCP_CUDA(cudaMalloc(&recv_counts, sizeof(int64_t) * P));
  HPCP_CUDA(cudaMalloc(&verdict, sizeof *verdict));
  HPCP_CUDA(cudaMalloc(&count, sizeof *count));
  cudaEvent_t e0, e1;
  HPCP_CUDA(cudaEventCreate(&e0));
  HPCP_CUDA(cudaEventCreate(&e1));
  uint32_t barrier_epoch = 0, ticket_issued = 0, it_global = 0;
  const bool memcpy_shape = cfg.stock == "memcpy";

  for (const size_t B : block_sizes(cfg)) {
    const int64_t mean = mean_rows(B, rb), cap = capacity_rows(P, mean);
    Row best;
    best.block_bytes = B;
    best.ms = std::numeric_limits<double>::max();
    std::vector<int64_t> m;
    for (int it = 0; it < cfg.warmup + cfg.iters; ++it, ++it_global) {
      NvtxRange range(it < cfg.warmup ? "alltoallv warm-up" : "alltoallv timed");
      m = draw_counts(cfg.counts, P, mean, it_global);
      const int64_t total = rows_into(m, P, me);
      // The rows the exchange touches are filled last, as the equal-block path does, so that the unused tail does not
      // hold the L2 when the timed region starts.
      launch_fill_pattern(reinterpret_cast<uint32_t*>(my_recv + total * rb), (cap - total) * rb / 4, kTailPoisonSeed,
                          stream);
      for (int q = 0; q < P; ++q)
        launch_fill_pattern(reinterpret_cast<uint32_t*>(my_send + a2av_send_offset(m.data(), P, me, q) * rb),
                            m[me * P + q] * rb / 4, pair_seed(it_global, me, q), stream);
      launch_fill_pattern(reinterpret_cast<uint32_t*>(my_recv), total * rb / 4, kPoisonSeed, stream);
      HPCP_CUDA(cudaMemcpyAsync(my_counts, m.data() + me * P, sizeof(int64_t) * P, cudaMemcpyHostToDevice, stream));
      HPCP_CUDA(cudaMemsetAsync(recv_counts, 0xFF, sizeof(int64_t) * P, stream));
      HPCP_CUDA(cudaMemsetAsync(verdict, 0xFF, sizeof *verdict, stream));
      HPCP_CUDA(cudaStreamSynchronize(stream));
      ctx.barrier();
      launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
      HPCP_CUDA(cudaEventRecord(e0, stream));
      int ctas = 0;
      if (memcpy_shape) {  // what a design that synchronised the host for the counts does after paying for it
        for (int j = 0; j < P; ++j) {
          const int p = (me + 1 + j) % P;
          const size_t n = m[me * P + p] * rb;
          if (n == 0) continue;
          HPCP_CUDA(cudaMemcpyAsync(static_cast<unsigned char*>(sh.recv.ptr[p]) + a2av_recv_offset(m.data(), P, me, p) * rb,
                                    my_send + a2av_send_offset(m.data(), P, me, p) * rb, n, cudaMemcpyDefault, stream));
        }
        launch_barrier_all(pads.data(), me, P, ++barrier_epoch, cfg.timeout_ns, status, stream);
      } else {
        AllToAllVArgs a;
        for (int r = 0; r < P; ++r) {
          a.send[r] = sh.send.ptr[r];
          a.recv[r] = sh.recv.ptr[r];
          a.counts[r] = static_cast<const int64_t*>(sh.counts.ptr[r]);
          a.pads[r] = pads[r];
        }
        a.recv_counts = recv_counts;
        a.verdict = verdict;
        a.ticket = my_pad + kPadLocal;
        a.ticket_base = ticket_issued;
        a.rank = me;
        a.world = P;
        a.row_bytes = rb;
        a.send_capacity_rows = cap;
        a.recv_capacity_rows = cap;
        a.barrier_epoch = ++barrier_epoch;
        a.timeout_ns = cfg.timeout_ns;
        a.status = status;
        a.pull = cfg.pull;
        ctas = launch_all_to_all_v(a, cfg.ctas, dev, stream);
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
      if (it >= cfg.warmup && t < best.ms) {
        best.ms = t;
        best.ctas = ctas;
        count_traffic(m, P, rb, best);
      }
    }
    // Every segment from p at its packed row against the seed of (p, me) in the last iteration; the rows past the
    // total still the poison; recv_counts and the verdict as the host's matrix says.
    const int64_t total = rows_into(m, P, me);
    HPCP_CUDA(cudaMemsetAsync(count, 0, sizeof *count, stream));
    for (int p = 0; p < P; ++p)
      launch_verify_pattern(reinterpret_cast<const uint32_t*>(my_recv + a2av_recv_offset(m.data(), P, p, me) * rb),
                            m[p * P + me] * rb / 4, pair_seed(it_global - 1, p, me), count, nullptr, nullptr, 0, 0,
                            nullptr, stream);
    launch_verify_pattern(reinterpret_cast<const uint32_t*>(my_recv + total * rb), (cap - total) * rb / 4,
                          kTailPoisonSeed, count, nullptr, nullptr, 0, 0, nullptr, stream);
    unsigned long long bad = 0;
    std::vector<int64_t> rc(P);
    uint32_t v = 0;
    HPCP_CUDA(cudaMemcpyAsync(&bad, count, sizeof bad, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaMemcpyAsync(rc.data(), recv_counts, sizeof(int64_t) * P, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaMemcpyAsync(&v, verdict, sizeof v, cudaMemcpyDeviceToHost, stream));
    HPCP_CUDA(cudaStreamSynchronize(stream));
    if (!memcpy_shape) {
      for (int p = 0; p < P; ++p) bad += rc[p] != m[p * P + me];
      bad += v != kA2avAccepted;
    }
    best.bad = static_cast<unsigned long long>(ctx.sum(static_cast<double>(bad)));
    print_verdict(me, bad);
    if (me == 0) sh.rows.push_back(best);
    ctx.barrier();
    if (me == 0) report_v(cfg, P, sh.rows.back());
    ctx.barrier();
  }
  (void)cudaFree(recv_counts);
  (void)cudaFree(verdict);
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
    send[me].resize((cfg.gather ? 1 : P) * top / 4);
    recv[me].resize(P * top / 4);
    uint32_t it_global = 0;
    for (const size_t B : sizes) {
      const size_t words = B / 4;
      double best_ms = std::numeric_limits<double>::max();
      for (int it = 0; it < cfg.warmup + cfg.iters; ++it, ++it_global) {
        if (cfg.gather)
          for (size_t i = 0; i < words; ++i) send[me][i] = pattern_word(i, gather_seed(it_global, me));
        else
          for (int q = 0; q < P; ++q)
            for (size_t i = 0; i < words; ++i) send[me][q * words + i] = pattern_word(i, pair_seed(it_global, me, q));
        for (size_t i = 0; i < P * words; ++i) recv[me][i] = pattern_word(i, kPoisonSeed);
        ctx.barrier();
        const auto t0 = std::chrono::steady_clock::now();
        for (int j = 0; j < P; ++j) {
          const int p = (me + 1 + j) % P;
          std::memcpy(recv[p].data() + me * words, send[me].data() + (cfg.gather ? 0 : p * words), B);
        }
        ctx.barrier();
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        const double t = ctx.max(ms);
        if (it >= cfg.warmup) best_ms = std::min(best_ms, t);
      }
      unsigned long long bad = 0;
      for (int p = 0; p < P; ++p) {
        const uint32_t seed = cfg.gather ? gather_seed(it_global - 1, p) : pair_seed(it_global - 1, p, me);
        for (size_t i = 0; i < words; ++i) bad += recv[me][p * words + i] != pattern_word(i, seed);
      }
      if (cfg.gather)
        for (size_t i = 0; i < words; ++i) bad += send[me][i] != pattern_word(i, gather_seed(it_global - 1, me));
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

// --counts without a GPU: the kernel's steps on host threads with the same plan rules (alltoallv_plan.h): the verdict,
// recv_counts, then the staggered walk of the packed segments as memcpy, then a barrier.
int run_on_host_v(const Config& cfg) {
  const int P = cfg.ranks;
  const size_t rb = cfg.row_bytes, rw = rb / 4;
  const std::vector<size_t> sizes = block_sizes(cfg);
  const int64_t top = capacity_rows(P, mean_rows(*std::max_element(sizes.begin(), sizes.end()), rb));
  std::vector<std::vector<uint32_t>> send(P), recv(P);
  std::vector<std::vector<int64_t>> recv_counts(P, std::vector<int64_t>(P));
  std::vector<Row> rows;
  run_ranks(P, [&](RankCtx& ctx) {
    const int me = ctx.rank;
    send[me].resize(top * rw);
    recv[me].resize(top * rw);
    uint32_t it_global = 0;
    for (const size_t B : sizes) {
      const int64_t mean = mean_rows(B, rb), cap = capacity_rows(P, mean);
      Row best;
      best.block_bytes = B;
      best.ms = std::numeric_limits<double>::max();
      std::vector<int64_t> m;
      uint32_t v = 0;
      for (int it = 0; it < cfg.warmup + cfg.iters; ++it, ++it_global) {
        m = draw_counts(cfg.counts, P, mean, it_global);
        const int64_t total = rows_into(m, P, me);
        for (int q = 0; q < P; ++q) {
          uint32_t* seg = send[me].data() + a2av_send_offset(m.data(), P, me, q) * rw;
          for (size_t i = 0; i < m[me * P + q] * rw; ++i) seg[i] = pattern_word(i, pair_seed(it_global, me, q));
        }
        for (size_t i = 0; i < total * rw; ++i) recv[me][i] = pattern_word(i, kPoisonSeed);
        for (size_t i = 0; i < (cap - total) * rw; ++i) recv[me][total * rw + i] = pattern_word(i, kTailPoisonSeed);
        std::fill(recv_counts[me].begin(), recv_counts[me].end(), -1);
        ctx.barrier();
        const auto t0 = std::chrono::steady_clock::now();
        v = a2av_verdict(m.data(), P, cap, cap);
        for (int p = 0; p < P; ++p) recv_counts[me][p] = m[p * P + me];
        if (v == kA2avAccepted)
          for (int j = 0; j < P; ++j) {
            const int p = (me + 1 + j) % P;
            std::memcpy(recv[p].data() + a2av_recv_offset(m.data(), P, me, p) * rw,
                        send[me].data() + a2av_send_offset(m.data(), P, me, p) * rw, m[me * P + p] * rb);
          }
        ctx.barrier();
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        const double t = ctx.max(ms);
        if (it >= cfg.warmup && t < best.ms) {
          best.ms = t;
          count_traffic(m, P, rb, best);
        }
      }
      const int64_t total = rows_into(m, P, me);
      unsigned long long bad = v != kA2avAccepted;
      for (int p = 0; p < P; ++p) {
        const uint32_t seed = pair_seed(it_global - 1, p, me);
        const uint32_t* seg = recv[me].data() + a2av_recv_offset(m.data(), P, p, me) * rw;
        for (size_t i = 0; i < m[p * P + me] * rw; ++i) bad += seg[i] != pattern_word(i, seed);
        bad += recv_counts[me][p] != m[p * P + me];
      }
      for (size_t i = 0; i < (cap - total) * rw; ++i) bad += recv[me][total * rw + i] != pattern_word(i, kTailPoisonSeed);
      best.bad = static_cast<unsigned long long>(ctx.sum(static_cast<double>(bad)));
      print_verdict(me, bad);
      if (me == 0) rows.push_back(best);
      ctx.barrier();
      if (me == 0) report_v(cfg, P, rows.back());
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
    {
      const std::string prog = argv[0];
      cfg.gather = prog.substr(prog.find_last_of('/') + 1) == "allgather";
    }
    static const option long_opts[] = {{"block-bytes", required_argument, nullptr, 1},
                                       {"pull", no_argument, nullptr, 2},
                                       {"stock", required_argument, nullptr, 3},
                                       {"sweep", no_argument, nullptr, 4},
                                       {"iters", required_argument, nullptr, 5},
                                       {"warmup", required_argument, nullptr, 6},
                                       {"ctas", required_argument, nullptr, 7},
                                       {"json", required_argument, nullptr, 8},
                                       {"cpu", no_argument, nullptr, 9},
                                       {"counts", required_argument, nullptr, 10},
                                       {"row-bytes", required_argument, nullptr, 11},
                                       {"help", no_argument, nullptr, 'h'},
                                       {nullptr, 0, nullptr, 0}};
    int opt;
    while ((opt = getopt_long(argc, argv, "hn:", long_opts, nullptr)) != -1) {
      switch (opt) {
        case 'h': print_help(cfg.gather); return 0;
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
        case 10: cfg.counts = optarg; break;
        case 11: {
          char* end = nullptr;
          cfg.row_bytes = std::strtoull(optarg, &end, 10);
          HPCP_REQUIRE(end != optarg && *end == '\0' && optarg[0] != '-', std::string("--row-bytes: not a byte count: ") + optarg);
          cfg.row_given = true;
          break;
        }
        default: print_help(cfg.gather); return 1;
      }
    }
    // Usage errors, before anything is allocated.
    HPCP_REQUIRE(cfg.stock.empty() || cfg.stock == "memcpy", "--stock must be memcpy, not " + cfg.stock);
    HPCP_REQUIRE(cfg.stock.empty() || !cfg.pull, "--stock memcpy is refused with --pull: the stock shape has no pull");
    HPCP_REQUIRE(cfg.stock.empty() || !cfg.cpu, "--stock memcpy is a GPU baseline: --cpu runs the host walk only");
    if (cfg.cpu && cfg.ranks < 0) cfg.ranks = 4;
    HPCP_REQUIRE(cfg.counts.empty() || cfg.counts == "random" || cfg.counts == "skewed" || cfg.counts == "equal",
                 "--counts must be random, skewed or equal, not " + cfg.counts);
    HPCP_REQUIRE(!cfg.row_given || !cfg.counts.empty(), "--row-bytes needs --counts");
    HPCP_REQUIRE(!cfg.gather || (cfg.counts.empty() && !cfg.row_given),
                 "allgather: --counts and --row-bytes belong to the all-to-all-v (bin/alltoall)");
    if (cfg.gather) {
      if (const char* why = all_gather_refusal(cfg.ranks < 0 ? 1 : cfg.ranks, cfg.block_bytes)) HPCP_FAIL(why);
    } else if (const char* why = all_to_all_refusal(cfg.ranks < 0 ? 1 : cfg.ranks, cfg.block_bytes)) {
      HPCP_FAIL(why);
    }
    if (!cfg.counts.empty())
      if (const char* why = all_to_all_v_refusal(cfg.ranks < 0 ? 1 : cfg.ranks, cfg.row_bytes, 1, 1)) HPCP_FAIL(why);

    if (cfg.cpu) return cfg.counts.empty() ? run_on_host(cfg) : run_on_host_v(cfg);
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
    const size_t top = *std::max_element(sizes.begin(), sizes.end());
    const bool v = !cfg.counts.empty();
    const size_t bytes = v ? capacity_rows(P, mean_rows(top, cfg.row_bytes)) * cfg.row_bytes : top * P;
    sh.pads = mem.alloc_pads(0);
    sh.send = mem.alloc(cfg.gather ? top : bytes, AllocKind::kDevice, /*zero=*/false);
    sh.recv = mem.alloc(bytes, AllocKind::kDevice, /*zero=*/false);
    if (v) sh.counts = mem.alloc(sizeof(int64_t) * P, AllocKind::kDevice, /*zero=*/true);
    run_ranks(P, [&](RankCtx& ctx) { v ? rank_main_v(ctx, sh) : rank_main(ctx, sh); });
    if (v) mem.free(sh.counts);
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
