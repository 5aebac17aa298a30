// Fabric topology: links -> connectivity planes -> rank placement.
//
// Capability parity with p2p/topology.cpp of the reference, which walks Level-Zero
// Sysman fabric ports, groups the two endpoints of every physical Xe-Link into a
// set and greedily merges overlapping sets into "planes" (topology.cpp:50-89),
// then prints the planes or the k-th device id (:92-106) for tile_mapping.sh.
//
// H100 redesign: links come from NVML (NVLink state / remote device type / remote
// PCI id per link) with cudaDeviceGetP2PAttribute as a second source; an NVSwitch
// is modelled as one extra fabric node so that every GPU hanging off the switch
// complex lands in the same plane.  The clustering itself is a union-find over
// link endpoint sets and takes an injected provider, so it is testable on a
// GPU-less machine (HPCP_FAKE_TOPOLOGY).
#pragma once

#include <map>
#include <set>
#include <string>
#include <vector>

namespace hpcp {
namespace topo {

struct GpuInfo {
  int index = 0;            // ordinal in the enumeration used for planes (NVML / PCI order)
  std::string name;
  std::string uuid;
  std::string pci_bus_id;   // "00000000:1B:00.0"
  int numa_node = -1;
  int nvlinks_active = 0;
  int nvlinks_to_switch = 0;
  bool multicast = false;   // NVLS capable (filled by the CUDA provider when available)
};

// One physical (or logical) link: the set of endpoints it joins.  GPU endpoints
// are decimal ordinals ("0".."7"); anything else (e.g. "nvswitch") is a fabric node.
using LinkSet = std::set<std::string>;

struct Fabric {
  std::vector<GpuInfo> gpus;
  std::vector<LinkSet> links;
  std::string source;       // "nvml", "cuda-p2p", "fake"
  // Optional pairwise attributes (filled by the CUDA provider).
  std::map<std::pair<int, int>, int> p2p_access, p2p_atomics, p2p_perf_rank;
};

// Merge link sets that share an endpoint (transitively) and keep GPU endpoints only.
// Every GPU appears in exactly one plane; isolated GPUs form singleton planes.
// Planes are ordered by their smallest member; members ascending.
std::vector<std::vector<int>> merge_planes(int n_gpus, const std::vector<LinkSet>& links);

// Flattened plane order: pairs (2k, 2k+1) of the flattening share a plane whenever
// plane sizes are even — the property peer2pear relies on.
std::vector<int> flatten(const std::vector<std::vector<int>>& planes);

// Rank -> device policies (↔ p2p/tile_mapping.sh:9-20).
//   compact      : rank r -> device r % n                (neighbouring ranks on neighbouring GPUs)
//   spread       : ranks dealt round-robin over `n_domains` halves of the node
//                  (r -> (r % d) * (n/d) + (r / d) % (n/d)), pairs straddle domains
//   compact_plan : rank r -> flatten(planes)[r % n]       (pairs share a fabric plane)
int device_for_rank(const std::string& policy, int local_rank, int n_devices,
                    const std::vector<std::vector<int>>& planes, int n_domains = 2);

// Providers.  Each returns false (with `why`) when unavailable.
bool fabric_from_fake(const std::string& spec, Fabric* out, std::string* why);  // "8:0-1,2-3" or "8:switch"
bool fabric_from_nvml(Fabric* out, std::string* why);
// Tries $HPCP_FAKE_TOPOLOGY, then NVML, then (if compiled in) the CUDA P2P matrix.
bool discover_fabric(Fabric* out, std::string* why);

std::string to_json(const Fabric& f, const std::vector<std::vector<int>>& planes);

}  // namespace topo
}  // namespace hpcp
