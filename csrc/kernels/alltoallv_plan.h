// The rules of the all-to-all-v (all_to_all_v_kernel in all_to_all.cu) as plain functions, shared by the kernel, the
// host walk of bin/alltoall --cpu and the bindings (tests/test_alltoallv_plan.py checks them against brute force, and
// the emulated device of tests/alltoallv_emu.py runs on them).
//
// The count matrix is row-major: m[p * world + q] = M[p][q], the rows rank p sends to rank q (int64, the unit of
// torch's split sizes).  Send and receive buffers are packed as in all_to_all_single: rank p's segment for q starts
// at row sum_{q' < q} M[p][q'] of its send buffer and lands at row sum_{p' < p} M[p'][q] of q's receive buffer.
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define HPCP_A2AV_HD __host__ __device__ __forceinline__
#else
#define HPCP_A2AV_HD inline
#endif

namespace hpcp {

// The verdict of a count matrix: 0 accepts it, otherwise the number of the first broken rule in this order.
enum AllToAllVVerdict : uint32_t {
  kA2avAccepted = 0,
  kA2avNegative = 1,      // some M[p][q] < 0
  kA2avSendCapacity = 2,  // some M[p][q], or some row sum, above send_capacity_rows
  kA2avRecvCapacity = 3,  // some column sum above recv_capacity_rows
};

// Rule of row p alone: kA2avNegative, kA2avSendCapacity or kA2avAccepted.  A count is compared with what is left of
// the capacity, so no sum ever exceeds the capacity and none can overflow.
HPCP_A2AV_HD uint32_t a2av_row_rule(const int64_t* m, int world, int p, int64_t send_capacity_rows) {
  uint32_t rule = kA2avAccepted;
  int64_t sum = 0;
  for (int q = 0; q < world; ++q) {
    const int64_t c = m[p * world + q];
    if (c < 0) return kA2avNegative;
    if (rule == kA2avAccepted && c > send_capacity_rows - sum) rule = kA2avSendCapacity;
    if (rule == kA2avAccepted) sum += c;
  }
  return rule;
}

// Rule of column q alone: kA2avRecvCapacity or kA2avAccepted.  Negative counts are left to the row rule, which wins.
HPCP_A2AV_HD uint32_t a2av_col_rule(const int64_t* m, int world, int q, int64_t recv_capacity_rows) {
  int64_t sum = 0;
  for (int p = 0; p < world; ++p) {
    const int64_t c = m[p * world + q];
    if (c < 0) continue;
    if (c > recv_capacity_rows - sum) return kA2avRecvCapacity;
    sum += c;
  }
  return kA2avAccepted;
}

// `broken` has bit k set when rule k is broken by some row or column (bit 0, "accepted", is ignored): the lowest rule.
HPCP_A2AV_HD uint32_t a2av_first_rule(uint32_t broken) {
  for (uint32_t k = kA2avNegative; k <= kA2avRecvCapacity; ++k)
    if (broken & (1u << k)) return k;
  return kA2avAccepted;
}

// The verdict of the whole world x world matrix (every rank computes the same one from the same matrix).
HPCP_A2AV_HD uint32_t a2av_verdict(const int64_t* m, int world, int64_t send_capacity_rows,
                                   int64_t recv_capacity_rows) {
  uint32_t broken = 0;
  for (int i = 0; i < world; ++i) {
    broken |= 1u << a2av_row_rule(m, world, i, send_capacity_rows);
    broken |= 1u << a2av_col_rule(m, world, i, recv_capacity_rows);
  }
  return a2av_first_rule(broken);
}

// Row of p's send buffer where its segment for q starts (an accepted matrix).
HPCP_A2AV_HD int64_t a2av_send_offset(const int64_t* m, int world, int p, int q) {
  int64_t off = 0;
  for (int j = 0; j < q; ++j) off += m[p * world + j];
  return off;
}

// Row of r's receive buffer where the segment from p starts (an accepted matrix).
HPCP_A2AV_HD int64_t a2av_recv_offset(const int64_t* m, int world, int p, int r) {
  int64_t off = 0;
  for (int j = 0; j < p; ++j) off += m[j * world + r];
  return off;
}

}  // namespace hpcp
