// blance_b200/csrc/schedule.cuh — the orchestrator's whole schedule under the lock-step model of
// include/blance_b200.h (blance_moves_schedule): rounds of findAvailableMovesUnlocked (orchestrate.go:749-763)
// followed, per node, by filterNextPlausibleMovesForNode (orchestrate.go:482-504) with
// LowestWeightPartitionMoveForNode (orchestrate.go:177-186).
//
// One round is a fixed sequence of launches that never waits for the host:
//   k_sched_keys   node of each active partition's next move (the sort key) and the per-node list lengths
//   radix sort     stable over ceil(log2(n_node_ids + 1)) key bits: per-node lists in ascending partition index
//   k_sched_scan   one CTA: list offsets and batch offsets over the nodes, the round's slice of round_off
//   k_sched_pick   one warp per non-empty node: the count picks with swap-remove, cursors advanced
//   k_sched_flags  + select: the active list compacted in order (finished and stuck partitions dropped)
// Every kernel reads the active count and the done flag from SchedState, so the host can enqueue a block of
// rounds and look at the flag once per block.  The work of a round is proportional to the bound on the active
// entries the host last read, plus n_node_ids for the scan - never to n_parts.  The schedules of a scenario wave
// (blance_plan_scenarios_schedule) run on wave_schedule.cuh instead, which shares the picks (sched_pick_node) but
// keeps the per-node lists between rounds rather than sorting every active entry each round.
#pragma once

#include <cuda_runtime.h>
#include <climits>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "aux_kernels.cuh"
#include "blance_b200.h"

namespace blance_dev {

struct SchedState {
  int32_t A;                 // active partitions (next < len and the next move's node has a mover)
  int32_t done;              // set by the first round that finds no active partition
  int32_t rounds;            // R so far
  int32_t max_batch;
  long long base;            // round_off[r] of the round in flight
  unsigned long long stuck;  // partitions dropped because their next move's node has no mover
};

__device__ __forceinline__ bool sched_pickable(int32_t node, int32_t n_node_ids, const uint8_t* __restrict__ mover) {
  return node >= 0 && node < n_node_ids && mover[node] != 0;
}

// cursors at 0, the candidate list = every partition (the first compaction filters it)
__global__ void k_sched_init(int32_t n_parts, int32_t* __restrict__ cur, int32_t* __restrict__ act,
                             long long* __restrict__ round_off, SchedState* st) {
  for (int32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_parts; p += gridDim.x * blockDim.x) {
    cur[p] = 0;
    act[p] = p;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    st->A = n_parts; st->done = 0; st->rounds = 0; st->max_batch = 0; st->base = 0; st->stuck = 0;
    round_off[0] = 0;
  }
}

// flags[i] = partition act[i] (i < A) still has a pickable next move.  One whose next move sits on a node without
// a mover can never advance (model rule 5): it is counted once here and leaves the active list for good.
__global__ void k_sched_flags(int32_t a_bound, const int32_t* __restrict__ act, const long long* __restrict__ off,
                              const int32_t* __restrict__ op_node, const int32_t* __restrict__ cur,
                              const uint8_t* __restrict__ mover, int32_t n_node_ids, uint8_t* __restrict__ flags,
                              SchedState* st) {
  const int32_t A = st->A;
  uint32_t stuck = 0;
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a_bound; i += gridDim.x * blockDim.x) {
    uint8_t f = 0;
    if (i < A) {
      const int32_t p = act[i];
      const long long o = off[p], c = cur[p];
      if (o + c < off[p + 1]) {
        if (sched_pickable(op_node[o + c], n_node_ids, mover)) f = 1;
        else ++stuck;
      }
    }
    flags[i] = f;
  }
  stuck = __reduce_add_sync(0xFFFFFFFFu, stuck);
  if ((threadIdx.x & 31) == 0 && stuck) atomicAdd(&st->stuck, (unsigned long long)stuck);
}

// sort key of each active entry = the node of its next move (n_node_ids past the active count: sorts last);
// cnt[node] = that node's list length
__global__ void k_sched_keys(int32_t a_bound, const int32_t* __restrict__ act, const long long* __restrict__ off,
                             const int32_t* __restrict__ op_node, const int32_t* __restrict__ cur, int32_t n_node_ids,
                             uint32_t* __restrict__ key, int32_t* __restrict__ cnt, const SchedState* st) {
  const int32_t A = st->A;
  for (int32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a_bound; i += gridDim.x * blockDim.x) {
    uint32_t k = (uint32_t)n_node_ids;
    if (i < A) {
      const int32_t p = act[i];
      const int32_t node = op_node[off[p] + cur[p]];
      k = (uint32_t)node;
      atomicAdd(&cnt[node], 1);
    }
    key[i] = k;
  }
}

// One CTA: noff = exclusive scan of the list lengths, boff = exclusive scan of the batch sizes min(count, length);
// the round's ops are round_off[r] + boff[n] ..; cnt is cleared for the next round.  A round that finds no active
// partition ends the schedule.
constexpr int SCHED_SCAN_THREADS = 512;             // 1024 threads cap the registers at 64: the int2 scan then spills

__global__ void __launch_bounds__(SCHED_SCAN_THREADS) k_sched_scan(int32_t n_node_ids, int32_t count, int32_t* __restrict__ cnt,
                                                                   int32_t* __restrict__ noff, int32_t* __restrict__ boff,
                                                                   long long* __restrict__ round_off, SchedState* st) {
  using Scan = cub::BlockScan<int2, SCHED_SCAN_THREADS>;
  using Reduce = cub::BlockReduce<int32_t, SCHED_SCAN_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ typename Reduce::TempStorage red_tmp;
  __shared__ int2 carry;
  if (st->done) return;
  if (st->A == 0) {
    if (threadIdx.x == 0) st->done = 1;
    return;
  }
  if (threadIdx.x == 0) carry = make_int2(0, 0);
  int32_t biggest = 0;
  for (int32_t base = 0; base < n_node_ids; base += SCHED_SCAN_THREADS) {
    const int32_t n = base + (int32_t)threadIdx.x;
    const int32_t len = n < n_node_ids ? cnt[n] : 0;
    const int32_t b = len < count ? len : count;
    biggest = b > biggest ? b : biggest;
    int2 excl, total;
    __syncthreads();                                   // carry of the previous chunk is visible, scan_tmp free
    Scan(scan_tmp).ExclusiveScan(make_int2(len, b), excl, make_int2(0, 0),
                                 [](const int2& x, const int2& y) { return make_int2(x.x + y.x, x.y + y.y); }, total);
    const int2 c = carry;
    if (n < n_node_ids) {
      noff[n] = c.x + excl.x;
      boff[n] = c.y + excl.y;
      cnt[n] = 0;
    }
    __syncthreads();                                   // everyone has read carry
    if (threadIdx.x == 0) carry = make_int2(c.x + total.x, c.y + total.y);
  }
  __syncthreads();
  const int32_t mx = Reduce(red_tmp).Reduce(biggest, cub::Max());
  if (threadIdx.x == 0) {
    noff[n_node_ids] = carry.x;
    boff[n_node_ids] = carry.y;
    const int32_t r = st->rounds;
    const long long b0 = round_off[r];
    st->base = b0;
    round_off[r + 1] = b0 + carry.y;
    st->rounds = r + 1;
    if (mx > st->max_batch) st->max_batch = mx;
  }
}

// filterNextPlausibleMovesForNode over one node's list of m entries, run by one warp: k picks, each the FIRST index
// of the minimal MoveOpWeight over the list as it stands (a warp arg-min of (weight, index)).  weight(i) reads entry
// i's weight; lane 0 calls take(j, i, last) for pick j at index i, and take must replace entry i by entry `last`
// (the swap-remove; the list then shrinks by one).  Lists of any length and counts up to the length are exact:
// every pick scans the whole remaining list.
template <class Weight, class Take>
__device__ __forceinline__ void sched_pick_node(int32_t m, int32_t k, int lane, Weight&& weight, Take&& take) {
  for (int32_t j = 0; j < k; ++j) {
    uint32_t bw = 8, bi = 0xFFFFFFFFu;
    for (int32_t i = lane; i < m; i += 32) {            // ascending i: the strict < keeps this lane's first minimum
      const uint32_t w = weight(i);
      if (w < bw) { bw = w; bi = (uint32_t)i; }
    }
    const uint32_t wmin = __reduce_min_sync(0xFFFFFFFFu, bw);
    const int32_t imin = (int32_t)__reduce_min_sync(0xFFFFFFFFu, bw == wmin ? bi : 0xFFFFFFFFu);
    if (lane == 0) take(j, imin, m - 1);
    __syncwarp();
    --m;
  }
}

// One warp per node: sched_pick_node over the node's list L (ascending partition index).  wl holds the weights
// next to L so that the scans touch two arrays only.
constexpr int SCHED_PICK_THREADS = 256;

__global__ void __launch_bounds__(SCHED_PICK_THREADS) k_sched_pick(int32_t n_node_ids, int32_t count,
                                                                   const int32_t* __restrict__ noff,
                                                                   const int32_t* __restrict__ boff, int32_t* __restrict__ list,
                                                                   uint8_t* __restrict__ wl, const long long* __restrict__ off,
                                                                   const uint8_t* __restrict__ op_kind, int32_t* __restrict__ cur,
                                                                   long long* __restrict__ sched_op, const SchedState* st) {
  if (st->done) return;
  const int lane = threadIdx.x & 31;
  const int32_t n_warps = (int32_t)(gridDim.x * (blockDim.x >> 5));
  const long long base = st->base;
  for (int32_t n = (int32_t)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); n < n_node_ids; n += n_warps) {
    const int32_t lo = noff[n];
    int32_t m = noff[n + 1] - lo;
    if (m == 0) continue;
    int32_t* L = list + lo;
    uint8_t* W = wl + lo;
    for (int32_t i = lane; i < m; i += 32) {
      const int32_t p = L[i];
      W[i] = (uint8_t)move_op_weight(op_kind[off[p] + cur[p]]);
    }
    __syncwarp();
    const int32_t k = m < count ? m : count;
    long long* out = sched_op + base + boff[n];
    sched_pick_node(m, k, lane, [&](int32_t i) { return (uint32_t)W[i]; }, [&](int32_t j, int32_t imin, int32_t last) {
      const int32_t p = L[imin];
      out[j] = off[p] + cur[p];
      cur[p] += 1;
      L[imin] = L[last];
      W[imin] = W[last];
    });
  }
}

}  // namespace blance_dev
