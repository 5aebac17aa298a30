// Host-only self-test of the native runtime pieces that need no GPU: the thread-per-rank runtime,
// the device-subset policy, the dtype trait table, plane clustering and rank->device policies, and
// the concurrency driver's pure functions.  Built as bin/native_selftest; run by tests/test_native_selftest.py
// (the reference has no unit tests at all).
#include <atomic>
#include <cstdint>
#include <cmath>
#include <cstdio>
#include <iostream>
#include <stdexcept>
#include <string>
#include <set>
#include <utility>
#include <vector>

#include "../common/dtype_traits.h"
#include "../common/rank_runtime.h"
#include "../concurency/driver.hpp"
#include "../kernels/alltoallv_plan.h"
#include "../kernels/ring_order.h"
#include "../kernels/tile_order.h"
#include "../miniapps/devices.hpp"
#include "../p2p/topology_core.hpp"

namespace {

int failures = 0;
#define CHECK(cond)                                                              \
  do {                                                                           \
    if (!(cond)) {                                                               \
      ++failures;                                                                \
      std::fprintf(stderr, "CHECK failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); \
    }                                                                            \
  } while (0)

void test_rank_runtime() {
  using namespace hpcp;
  for (int world : {1, 2, 8}) {
    std::atomic<int> visited{0};
    std::vector<double> maxes(world), mins(world), sums(world);
    run_ranks(world, [&](RankCtx& ctx) {
      CHECK(ctx.world == world);
      for (int it = 0; it < 50; ++it) {
        ctx.barrier();
        maxes[ctx.rank] = ctx.max(static_cast<double>(ctx.rank * 10 + it));
        mins[ctx.rank] = ctx.min(static_cast<double>(ctx.rank + it));
        sums[ctx.rank] = ctx.sum(1.0);
      }
      visited.fetch_add(1);
    });
    CHECK(visited.load() == world);
    for (int r = 0; r < world; ++r) {
      CHECK(maxes[r] == (world - 1) * 10 + 49);
      CHECK(mins[r] == 49);
      CHECK(sums[r] == world);
    }
  }
  // A failing rank must not leave the others stuck in a barrier; the root cause is rethrown.
  bool threw = false;
  try {
    run_ranks(4, [&](RankCtx& ctx) {
      if (ctx.rank == 2) throw std::runtime_error("rank 2 exploded");
      ctx.barrier();
      ctx.barrier();
    });
  } catch (const std::exception& e) {
    threw = std::string(e.what()) == "rank 2 exploded";
  }
  CHECK(threw);
}

void test_devices_and_dtypes() {
  using namespace hpcp;
  CHECK(device_subset(3, 8, 8) == std::vector<int>({3}));
  CHECK(device_subset(1, 4, 8) == std::vector<int>({2, 3}));        // contiguous block of ndev/size
  CHECK(device_subset(5, 8, 2) == std::vector<int>({1}));           // oversubscription: round-robin
  CHECK(device_subset(0, 4, 0).empty());
  CHECK(primary_device(5, 8, 2) == 1);
  CHECK(primary_device(1, 4, 8) == 3);                               // subset {2,3}[1 % 2]
  CHECK(primary_device(0, 1, 0) == -1);
  CHECK(std::string(get_dtype<float>().name) == "float" && get_dtype<float>().reducible);
  CHECK(std::string(get_dtype<int>().name) == "int" && get_dtype<int>().elem == ElemType::kInt);
  // every type the reference's trait maps to an MPI_SUM datatype (mpi_datatype.hpp:28-51) reduces here too
  CHECK(get_dtype<double>().reducible && get_dtype<double>().size == 8 && get_dtype<double>().elem == ElemType::kDouble);
  CHECK(get_dtype<long>().reducible && get_dtype<long>().elem == ElemType::kLong && elem_size(ElemType::kLong) == 8);
  CHECK(get_dtype<unsigned short>().elem == ElemType::kUShort && elem_size(ElemType::kUShort) == 2);
  CHECK(get_dtype<unsigned char>().reducible && elem_size(ElemType::kUChar) == 1);
  CHECK(!get_dtype<long double>().reducible);                      // no device representation: bytes
  struct Opaque { char x[24]; };
  CHECK(std::string(get_dtype<Opaque>().name) == "bytes" && get_dtype<Opaque>().size == 24);  // MPI_BYTE analogue
  ElemType t;
  CHECK(elem_type_from_name("int32", &t) && t == ElemType::kInt);
  CHECK(elem_type_from_name("unsigned long", &t) && t == ElemType::kULong && std::string(elem_type_name(t)) == "ulong");
  CHECK(elem_type_from_name("float64", &t) && t == ElemType::kDouble);
  CHECK(!elem_type_from_name("complex", &t));
}

void test_topology() {
  using namespace hpcp::topo;
  Fabric f;
  std::string why;
  CHECK(fabric_from_fake("8:switch", &f, &why));
  auto planes = merge_planes(8, f.links);
  CHECK(planes.size() == 1 && planes[0].size() == 8);
  CHECK(fabric_from_fake("6:0-2,2-4,1-3,3-5", &f, &why));
  planes = merge_planes(6, f.links);
  CHECK(planes.size() == 2 && planes[0] == std::vector<int>({0, 2, 4}) && planes[1] == std::vector<int>({1, 3, 5}));
  CHECK(flatten(planes) == std::vector<int>({0, 2, 4, 1, 3, 5}));
  CHECK(device_for_rank("compact", 9, 8, planes) == 1);
  CHECK(device_for_rank("spread", 1, 8, planes) == 4);
  CHECK(device_for_rank("compact_plan", 3, 6, planes) == 1);
  bool threw = false;
  try {
    device_for_rank("diagonal", 0, 8, planes);
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  CHECK(threw);
  CHECK(!fabric_from_fake("nonsense", &f, &why));
  CHECK(to_json(f, planes).find("\"planes\":[[0,2,4],[1,3,5]]") != std::string::npos);
}

void test_driver_pure_functions() {
  using namespace hpcp::con;
  CHECK(strip_twos("M2D") == "MD" && strip_twos("22") == "");
  CHECK(is_compute_command("C") && is_compute_command("T") && !is_compute_command("MD"));
  CHECK(tuned_parameter_of("C") == "tripcount_C" && tuned_parameter_of("T") == "tripcount_T" &&
        tuned_parameter_of("DP") == "globalsize_DP");
  Params p{{"globalsize_MD", 250000000}, {"globalsize_C", 1}};
  CHECK(bytes_moved({"C", "MD"}, p, 4) == 1000000000ull);
  CHECK(bytes_moved({"MD", "MD", "MD", "MD", "MD"}, p, 4) == 5000000000ull);   // > 2^32: no wrap
  CHECK(time_with_bandwidth(1000, 0) == "1000us");
  CHECK(time_with_bandwidth(1000, 1000000) == "1000us (1 GBytes/s)");
  CHECK(judge(2.0, 1.9, 10, -1, 100) == Verdict::kSuccess);
  CHECK(judge(2.0, 1.5, 10, -1, 100) == Verdict::kFarFromTheoretical);          // 2.0 >= 1.3 * 1.5
  CHECK(judge(2.0, 2.0, 10, 50, 100) == Verdict::kBandwidthFloor);
  CHECK(verdict_line("fused", {"C", "DP"}, Verdict::kSuccess) ==
        "## fused | C DP | SUCCESS: Close from Theoretical Speedup");
  auto fake = make_fake_backend("C=0.01,MD=0.0005,overlap=1.0");
  bool usage = false;
  try {
    parse_arguments({"in_order", "--commands", "Q"}, *fake);
  } catch (const UsageError&) {
    usage = true;
  }
  CHECK(usage);
  const Options opt = parse_arguments({"fused", "--queues", "3", "--commands", "C", "M2D", "--commands", "D2P"}, *fake);
  CHECK(opt.mode == "fused" && opt.n_queues == 3 && opt.groups.size() == 2 && opt.groups[0][1] == "MD");
  Params params = resolve_parameters(opt);
  CHECK(params.at("tripcount_C") == 40000 && params.at("globalsize_C") == 1 &&
        params.at("globalsize_MD") == 250000000);
}

}  // namespace

// The orderings the tensor-core kernels and the ring kernel run on the device (host + device headers).
void test_kernel_orderings() {
  using namespace hpcp;
  using namespace hpcp::umma;
  for (int tiles_m : {1, 2, 7, 8, 16, 64})
    for (int tiles_n : {1, 3, 32}) {
      std::set<std::pair<int, int>> seen;
      for (int t = 0; t < tiles_m * tiles_n; ++t) {
        int mb = -1, nb = -1;
        tile_coords(t, tiles_m, tiles_n, &mb, &nb);
        CHECK(mb >= 0 && mb < tiles_m && nb >= 0 && nb < tiles_n);
        seen.insert({mb, nb});
      }
      CHECK(static_cast<int>(seen.size()) == tiles_m * tiles_n);  // a bijection
    }
  // Shard-major order: rank r starts with the shard of rank r + first; all ranks are on different shards at any time.
  const int world = 8, shard_tiles_m = 4, tiles_n = 3, per_shard = shard_tiles_m * tiles_n;
  for (int first : {0, 1})
    for (int t = 0; t < world * per_shard; t += 5) {
      std::set<int> owners;
      for (int r = 0; r < world; ++r) {
        int mb = 0, nb = 0;
        shard_coords(t, r, world, first, shard_tiles_m, tiles_n, &mb, &nb);
        CHECK(mb / shard_tiles_m == (r + first + t / per_shard) % world);
        owners.insert(mb / shard_tiles_m);
      }
      CHECK(static_cast<int>(owners.size()) == world);
    }
  // Gather pieces of the all-gather -> GEMM kernel: every remote byte exactly once, counted on the block it lands in.
  const uint32_t cpb = 8, chunk = 4096;
  const size_t block_bytes = static_cast<size_t>(cpb) * chunk;
  std::set<size_t> dst;
  for (size_t c = 0; c < static_cast<size_t>(world - 1) * shard_tiles_m * cpb; ++c) {
    const GatherPiece p = gather_piece(c, 3, world, shard_tiles_m, cpb, chunk, block_bytes);
    CHECK(p.peer != 3 && p.m_blk == static_cast<int>(p.dst_off / block_bytes));
    CHECK(p.dst_off == static_cast<size_t>(p.peer) * shard_tiles_m * block_bytes + p.src_off);
    dst.insert(p.dst_off);
  }
  CHECK(dst.size() == static_cast<size_t>(world - 1) * shard_tiles_m * cpb);
  // Ring slots and acks: every ack that is waited for is published, and nothing else.
  for (int P = 1; P <= 9; ++P)
    for (int t = 0; t < P; ++t) {
      if (t + 1 < P) CHECK(ring_waits_for_ack(t + 1, P) == ring_publishes_ack(t, P) || t == 0);
      CHECK(!ring_waits_for_ack(t, P) || (t >= 2 && ring_forwards(t, P)));
      CHECK(ring_src_slot(t + 1, true) == ring_fwd_slot(t, true));   // what hop t forwards is what hop t+1 reads
      CHECK(ring_src_slot(t + 1, false) == ring_fwd_slot(t, false));
    }
  // Reduce-scatter + all-gather ring: segment r is finished on rank r, every slot is written once and read by the next
  // hop, the all-gather never pushes into the right neighbour's own segment, and every publish is awaited.
  for (int P = 1; P <= 9; ++P)
    for (int phase : {int(kRsAgAllreduce), int(kRsAgReduceScatter), int(kRsAgAllGather)}) {
      const int first = rsag_first_hop(phase, P), last = rsag_last_hop(phase, P);
      CHECK(rsag_epoch_advance(phase, P) == (phase == kRsAgAllreduce ? 2 : 1) * (P - 1));
      CHECK(!rsag_waits(first, phase, P) && rsag_arrival(first, phase, P) == 0);
      std::set<int> slots_written;
      for (int h = first; h <= last; ++h)
        for (int r = 0; r < P; ++r) {
          const int seg = rsag_segment(h, r, P);
          CHECK(seg >= 0 && seg < P);
          CHECK(!rsag_writes_own_vc(h, P) || seg == r);
          CHECK(seg == rsag_segment(h - 1, (r - 1 + P) % P, P));  // the left neighbour's previous hop: same segment
          if (rsag_publishes(h, phase, P)) {
            CHECK(h < last && rsag_waits(h + 1, phase, P));
            CHECK(rsag_arrival(h + 1, phase, P) == rsag_arrival(h, phase, P) + 1);
            const int fs = rsag_fwd_slot(h, P);
            if (fs >= 0) {
              CHECK(rsag_src_slot(h + 1, phase, P) == fs);
              if (r == 0) CHECK(slots_written.insert(fs).second);
            } else {
              CHECK(seg != (r + 1) % P);
            }
          }
        }
      CHECK(static_cast<int>(slots_written.size()) == (phase == kRsAgAllGather ? 0 : P - 1));
    }
}

// All-to-all-v plan: on accepted matrices the receive segments of every rank tile [0, column sum) and the send
// segments [0, row sum) in order; the first broken rule wins.
void test_alltoallv_plan() {
  using namespace hpcp;
  uint64_t x = 0x9E3779B97F4A7C15ull;
  const auto next = [&x] { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
  for (int P = 1; P <= 16; ++P)
    for (int trial = 0; trial < 20; ++trial) {
      std::vector<int64_t> m(P * P);
      for (auto& c : m) c = static_cast<int64_t>(next() % 5);
      const int64_t cap = 4 * P;
      CHECK(a2av_verdict(m.data(), P, cap, cap) == kA2avAccepted);
      for (int r = 0; r < P; ++r) {
        int64_t rows = 0, sent = 0;
        for (int p = 0; p < P; ++p) {
          CHECK(a2av_recv_offset(m.data(), P, p, r) == rows);
          CHECK(a2av_send_offset(m.data(), P, r, p) == sent);
          rows += m[p * P + r];
          sent += m[r * P + p];
        }
        CHECK(rows <= cap && sent <= cap);
      }
      if (P > 1) {
        m[P + 1] = cap + 1;                                                      // one count above the send capacity
        CHECK(a2av_verdict(m.data(), P, cap, 1000 * cap) == kA2avSendCapacity);
        CHECK(a2av_verdict(m.data(), P, 1000 * cap, cap) == kA2avRecvCapacity);
        m[P * P - 1] = -1;                                                       // a negative beats every other rule
        CHECK(a2av_verdict(m.data(), P, cap, cap) == kA2avNegative);
      }
    }
  const int64_t big = INT64_MAX;                                                 // sums stop at the capacity: no overflow
  const int64_t m2[4] = {big, big, big, big};
  CHECK(a2av_verdict(m2, 2, big, big) == kA2avSendCapacity);
  CHECK(a2av_first_rule(0) == kA2avAccepted && a2av_first_rule(0xE) == kA2avNegative && a2av_first_rule(9) == kA2avRecvCapacity);
}

// The host refusals of the stand-alone reduce-scatter and all-gather (kernels/api.h), before any launch.
void test_gather_scatter_refusals() {
  using namespace hpcp;
  CHECK(reduce_scatter_refusal(4, 4, ElemType::kFloat) == nullptr);
  CHECK(reduce_scatter_refusal(1, 1, ElemType::kDoubleInt) == nullptr);         // one 16-byte pair is a whole vector
  CHECK(reduce_scatter_refusal(16, 16, ElemType::kUChar) == nullptr);
  CHECK(reduce_scatter_refusal(4, 0, ElemType::kFloat) == kReduceScatterCountError);
  CHECK(reduce_scatter_refusal(4, 3, ElemType::kFloat) == kReduceScatterCountError);
  CHECK(reduce_scatter_refusal(4, 4, ElemType::kBFloat16) == kReduceScatterCountError);   // 8 bytes
  CHECK(reduce_scatter_refusal(0, 4, ElemType::kFloat) == kReduceScatterWorldError);
  CHECK(reduce_scatter_refusal(17, 4, ElemType::kFloat) == kReduceScatterWorldError);
  CHECK(all_gather_refusal(1, 16) == nullptr && all_gather_refusal(16, 48) == nullptr);
  CHECK(all_gather_refusal(4, 0) == kAllGatherBlockError && all_gather_refusal(4, 24) == kAllGatherBlockError);
  CHECK(all_gather_refusal(0, 16) == kAllGatherWorldError && all_gather_refusal(17, 16) == kAllGatherWorldError);
  alignas(16) static unsigned char buf[256];
  CHECK(byte_ranges_overlap(buf, 64, buf + 32, 16));                            // recv inside send (MPI_IN_PLACE)
  CHECK(byte_ranges_overlap(buf + 32, 16, buf, 64));
  CHECK(!byte_ranges_overlap(buf, 64, buf + 64, 64) && !byte_ranges_overlap(buf + 64, 64, buf, 64));
  CHECK(!reduce_op_takes(ReduceOp::kBAnd, ElemType::kHalf) && reduce_op_takes(ReduceOp::kBAnd, ElemType::kUShort));
}

int main() {
  test_kernel_orderings();
  test_alltoallv_plan();
  test_gather_scatter_refusals();
  test_rank_runtime();
  test_devices_and_dtypes();
  test_topology();
  test_driver_pure_functions();
  if (failures == 0) {
    std::cout << "native selftest: OK" << std::endl;
    return 0;
  }
  std::cout << "native selftest: " << failures << " failure(s)" << std::endl;
  return 1;
}
