// Slot and flow-control rules of the fused ring allreduce (ring_allreduce.cu) as plain functions, shared by
// the kernel and the host: tests/test_ring_protocol.py runs a randomly scheduled model of P ranks on top of
// exactly these rules and checks that no chunk is overwritten before its reader has consumed it.
//
// Hop t = 0 .. P-1 of a rank: read block `src` (t = 0: the rank's own VA, else receive slot ring_src_slot(t)),
// add it into VC and, unless it is the last hop, forward it into the right neighbour's slot ring_fwd_slot(t).
#pragma once

#if defined(__CUDACC__)
#define HPCP_RING_HD __host__ __device__ __forceinline__
#else
#define HPCP_RING_HD inline
#endif

namespace hpcp {

// two_slots = false: P-1 slots, hop t lands in slot t-1 (never reused inside one allreduce).
// two_slots = true : the reference's VA/VB double buffer, hop t lands in slot (t-1) % 2.
HPCP_RING_HD int ring_src_slot(int t, bool two_slots) { return two_slots ? ((t - 1) & 1) : t - 1; }
HPCP_RING_HD int ring_fwd_slot(int t, bool two_slots) { return two_slots ? (t & 1) : t; }
HPCP_RING_HD bool ring_forwards(int t, int world) { return t < world - 1; }
// Two slots: the forward of hop t >= 2 overwrites what the right neighbour reads at ITS hop t-1, so the sender
// first waits for the neighbour's ack of hop t-1 ...
HPCP_RING_HD bool ring_waits_for_ack(int t, int world) { return t >= 2 && ring_forwards(t, world); }
// ... and a receiver acks exactly the hops whose slot will be written again (by the sender's hop t+1).
HPCP_RING_HD bool ring_publishes_ack(int t, int world) { return t >= 1 && ring_waits_for_ack(t + 1, world); }

// ---- pull variant: a rank READS the block its left neighbour processed one hop earlier (NVLink loads), adds it and
// keeps a local copy for its right neighbour to read one hop later.  Hop 1 reads the neighbour's VA directly.
// Local copy of hop t (1 <= t <= P-2; the last hop is read by nobody): slot t-1, or (t-1) % 2 with two slots.
HPCP_RING_HD bool ring_pull_keeps_copy(int t, int world) { return t >= 1 && t <= world - 2; }
HPCP_RING_HD int ring_pull_copy_slot(int t, bool two_slots) { return two_slots ? ((t - 1) & 1) : t - 1; }
// Source of hop t >= 2 inside the LEFT neighbour's slots = the copy it kept at its hop t-1.
HPCP_RING_HD int ring_pull_src_slot(int t, bool two_slots) { return ring_pull_copy_slot(t - 1, two_slots); }
// Two slots: the copy of hop t overwrites the copy of hop t-2, which the right neighbour reads at ITS hop t-1 ...
HPCP_RING_HD bool ring_pull_waits_for_ack(int t, int world) { return t >= 3 && ring_pull_keeps_copy(t, world); }
// ... so a reader acks the hops whose source copy will be overwritten (by the owner's hop t+1).
HPCP_RING_HD bool ring_pull_publishes_ack(int t, int world) { return t >= 2 && ring_pull_waits_for_ack(t + 1, world); }

// ---- bandwidth-optimal ring (ring_rsag_kernel): reduce-scatter, then all-gather.  The block is P segments of whole
// 16-byte vectors; at hop h = 0 .. 2P-2 rank r works on segment rsag_segment(h, r, P) = (r - 1 - h) mod P:
//   h = 0          read own VA[seg]                          -> right's slot 0
//   1 <= h <= P-2  read slot h-1, add own VA[seg]            -> right's slot h
//   h = P-1        read slot P-2, add own VA[r] (seg == r)   -> own VC[r] and right's VC[r]
//   P <= h <= 2P-3 read own VC[seg] (the left neighbour put it there)   -> right's VC[seg]
//   h = 2P-2       only wait: VC[seg] is final
// Segment s is summed once, by rank s: ((VA[s+1] + VA[s+2]) + ...) + VA[s].  Every slot and every VC segment is written
// once per launch, so no ack channel is needed.  A phase runs part of the hops (rsag_first_hop .. rsag_last_hop); the
// all-gather starts at hop P-1 with VA[r] as its source.
enum RsAgPhase : int { kRsAgAllreduce = 0, kRsAgReduceScatter = 1, kRsAgAllGather = 2 };

HPCP_RING_HD int rsag_first_hop(int phase, int world) { return phase == kRsAgAllGather ? world - 1 : 0; }
HPCP_RING_HD int rsag_last_hop(int phase, int world) { return phase == kRsAgReduceScatter ? world - 1 : 2 * world - 2; }
HPCP_RING_HD int rsag_segment(int h, int rank, int world) { return ((rank - 1 - h) % world + world) % world; }
// Source of hop h: own VC[seg] from hop P on, else own VA[seg] ...
HPCP_RING_HD bool rsag_reads_vc(int h, int world) { return h >= world; }
// ... plus, at 1 <= h <= P-1 of a phase that reduces, receive slot h-1 (-1: none).
HPCP_RING_HD int rsag_src_slot(int h, int phase, int world) {
  return phase != kRsAgAllGather && h >= 1 && h <= world - 1 ? h - 1 : -1;
}
HPCP_RING_HD bool rsag_writes_own_vc(int h, int world) { return h == world - 1; }
// Push into the right neighbour: slot h while reducing, its VC[seg] from hop P-1 on (not in the reduce-scatter).
HPCP_RING_HD bool rsag_forwards(int h, int phase, int world) {
  return phase == kRsAgReduceScatter ? h <= world - 2 : h <= 2 * world - 3;
}
HPCP_RING_HD int rsag_fwd_slot(int h, int world) { return h <= world - 2 ? h : -1; }  // -1: the right's VC[seg]
HPCP_RING_HD bool rsag_waits(int h, int phase, int world) { return h > rsag_first_hop(phase, world); }
HPCP_RING_HD bool rsag_publishes(int h, int phase, int world) { return rsag_forwards(h, phase, world); }
// Arrival words count up from the launch's epoch base: hop h waits for base + rsag_arrival(h) and its push publishes
// base + rsag_arrival(h + 1).  A launch advances the base by rsag_epoch_advance: 2(P-1), P-1 per half.
HPCP_RING_HD int rsag_arrival(int h, int phase, int world) { return h - rsag_first_hop(phase, world); }
HPCP_RING_HD int rsag_epoch_advance(int phase, int world) {
  return rsag_arrival(rsag_last_hop(phase, world), phase, world);
}

}  // namespace hpcp
