// blance_b200/csrc/count_bound.hpp — the bound that keeps every node count of the pass kernels inside int32.
//
// The reference counts in Go's 64-bit int; the pass kernels keep a node's total as int32: the counts of the model
// states plus the counts of non-model states (extra_tot_first / extra_tot_rest), t = extra[n] + sum_s counts[s][n]
// (assign_pass*.cuh).  A partition adds its weight once per slot it holds a node in, so
//     sum_p |w_p| * max(1, n_slots) + max_n max(|extra_tot_first[n]|, |extra_tot_rest[n]|)
// bounds |t| and every count that makes it up, at every step of every iteration.  An instance whose bound is above
// INT32_MAX is BLANCE_ERR_UNSUPPORTED: blance_plan_in_check, the host interning and the scenario entry points (with
// each scenario's options applied) all check it here.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstdlib>

#include "blance_b200.h"

#define BLANCE_COUNT_BOUND_MSG "sum of |partition weight| x slots plus the largest non-model count exceeds int32 (the device keeps int32 counts)"

// sum over the partitions of |weight|, 1 for a partition without one (or when has_part_weights is 0)
inline long long count_bound_weight_sum(const blance_plan_in& in) {
  long long sum = 0;
  for (int32_t p = 0; p < in.n_parts; ++p)
    sum += in.has_part_weights && in.part_has_weight[p] ? std::llabs((long long)in.part_weight[p]) : 1;
  return sum;
}

// max over the nodes of |extra_tot_first[n]| and |extra_tot_rest[n]| (NULL arrays are zero)
inline long long count_bound_max_extra(int32_t n_nodes, const int32_t* extra_first, const int32_t* extra_rest) {
  long long m = 0;
  for (int32_t n = 0; n < n_nodes; ++n) {
    if (extra_first) m = std::max(m, std::llabs((long long)extra_first[n]));
    if (extra_rest) m = std::max(m, std::llabs((long long)extra_rest[n]));
  }
  return m;
}

// true when the counts fit int32.  weight_sum is at most 2^30 x 2^31, so it is tested alone before it is scaled.
inline bool count_bound_fits(long long weight_sum, int32_t n_slots, long long max_extra) {
  return weight_sum <= INT32_MAX && max_extra <= INT32_MAX &&
         weight_sum * std::max<long long>(1, n_slots) + max_extra <= INT32_MAX;
}

inline bool count_bound_fits(const blance_plan_in& in) {
  return count_bound_fits(count_bound_weight_sum(in), in.n_slots, count_bound_max_extra(in.n_nodes, in.extra_tot_first, in.extra_tot_rest));
}
