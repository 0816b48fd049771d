// blance_b200/csrc/wave_schedule.cuh — the lock-step schedule of include/blance_b200.h (blance_moves_schedule)
// for every scenario of a blance_plan_scenarios_schedule wave at once, reduced to per-node and per-partition
// summaries.
//
// An instance is a pair (scenario j of the wave, count index k): i = j * nc + k.  All instances run in lock step:
// global round r is round r of every instance that still has entries.  A segment is one (instance, node q) pair,
// s = i * NU + q.  The engine keeps, per segment, the list findAvailableMovesUnlocked builds (orchestrate.go:749-763):
// the partitions whose next op is on q, in ascending partition index, each entry (MoveOpWeight << 29) | p.  A
// partition has at most one op per node (CalcPartitionMoves' "seen" rule), so a segment never holds more entries
// than node_ops counts on its node: segment capacities are carved from the scenario summary.
//
// Between rounds a list changes only by its own picks leaving and by partitions arriving from picks elsewhere, so
// a round is a fixed launch sequence whose work follows the list entries and the round's picks:
//   scan           of the segments' pick counts min(count, length): each segment's slots for its arrival keys
//   k_wave_pick    one warp per non-empty segment: sched_pick_node (the picks of k_sched_pick), picked entries
//                  tombstoned (weight bits 0) in place, summaries and cursors updated, and the arrival key
//                  (segment of the next op << PB) | p written for every picked partition with a pickable next op
//   radix sort     of the round's arrival slots only (a host bound on the picks, padded with ~0)
//   k_wave_bounds  the slice of the sorted arrivals of each segment that received any
//   k_wave_merge   one warp per touched segment: survivors (in order) merged with its arrivals into the other list
//                  buffer, and its next pick count
// The lists are first built by the same sort, bounds and merge from the keys k_wave_moves writes for every
// partition's first op.  A round without picks changes nothing, so the host enqueues blocks of rounds and reads the
// last round's pick count once per block.
#pragma once

#include <cuda_runtime.h>

#include "aux_kernels.cuh"
#include "schedule.cuh"

namespace blance_dev {

constexpr int WAVE_PART_BITS = 29;                          // entry = (weight << 29) | partition; weight 0 = picked
constexpr uint32_t WAVE_PMASK = (1u << WAVE_PART_BITS) - 1;

struct WSched {
  int32_t nw, nc, PU, NU, MO, PB;          // scenarios, counts, partitions per scenario, node ids, ops per partition, key bits of p
  long long nseg;                          // nw * nc * NU
  const int32_t* count;                    // [nc] picks per node and round (max(1, MaxConcurrentPartitionMovesPerNode))
  const uint8_t* mover;                    // [NU]
  uint8_t* op_n; int32_t* op_node; uint8_t* op_w;    // [nw * PU], [nw * PU][MO]: ops of scenario j's partition p
  uint8_t* cur; int32_t* part_done;        // [ni * PU]: cursor, part_done_round
  const long long* seg_off;                // [nseg + 1] segment capacities carved from node_ops
  int32_t* len; int32_t* kcnt;             // [nseg + 1]: list length, picks of the next round (kcnt[nseg] = 0)
  const long long* poff;                   // [nseg + 1] exclusive scan of kcnt: arrival slots, poff[nseg] = picks
  int32_t* astart; int32_t* aend; int32_t* node_rounds; int32_t* node_last;   // [nseg]
  uint32_t* buf0; uint32_t* buf1; uint32_t* scratch;                          // [seg_off[nseg]]
  unsigned long long* keys_in; const unsigned long long* keys_out;             // arrival keys
  unsigned long long* scal;                // [ni][4]: rounds, moves_done, stuck_parts, max_batch
  int32_t* overflow;                       // more picks than the host sorted (internal error)
  long long* esum;                         // the host's reduction of len: entries left in all lists
};

__device__ __forceinline__ bool wave_pickable(const WSched& W, int32_t node) {
  return node >= 0 && node < W.NU && W.mover[node] != 0;
}

// CalcPartitionMoves of every assigned partition of every scenario (the rules of k_scenario_summary: the prev row as
// uploaded, an empty row for a partition absent from prevMap), then, per instance, the partition's first op: its
// arrival key in slot i * PU + p when the op's node has a mover, else the partition is stuck.  Grid: x strides over
// the partitions of scenario blockIdx.y.
__global__ void k_wave_moves(DPool pool, const int32_t* __restrict__ prev_rows_init, const uint8_t* __restrict__ pflags_init,
                             int32_t favor_min, WSched W) {
  const int j = blockIdx.y;
  const DInst& D = pool.insts[j];
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < D.PU; p += (long long)gridDim.x * blockDim.x) {
    const long long g = D.part_off + p;
    const long long gp = (long long)j * W.PU + p;
    const uint8_t f = pflags_init[g];
    int32_t* on = W.op_node + gp * W.MO;
    uint8_t* ow = W.op_w + gp * W.MO;
    int cnt = 0;
    if (f & PF_IN_ASSIGN) {
      auto emit = [&](int32_t node, int, int kind) {
        for (int x = 0; x < cnt; ++x) if (on[x] == node) return;   // addMoves + seen, moves.go:51-58
        on[cnt] = node; ow[cnt] = (uint8_t)move_op_weight(kind); ++cnt;
      };
      const int32_t* next = pool.rows + D.rows_off + p * D.SLP;
      if (f & PF_IN_PREV) calc_moves_row(prev_rows_init + D.rows_off + p * D.SLP, next, D.state_slot_off, D.SL, D.S, favor_min, emit);
      else {
        int32_t blank[BL_SLP_MAX];
        for (int c = 0; c < BL_SLP_MAX; ++c) blank[c] = BLANCE_NO_NODE;
        calc_moves_row(blank, next, D.state_slot_off, D.SL, D.S, favor_min, emit);
      }
    }
    W.op_n[gp] = (uint8_t)cnt;
    const bool pick0 = cnt > 0 && wave_pickable(W, on[0]);
    for (int k = 0; k < W.nc; ++k) {
      const long long i = (long long)j * W.nc + k;
      W.cur[i * W.PU + p] = 0;
      W.part_done[i * W.PU + p] = cnt == 0 || pick0 ? 0 : -1;
      W.keys_in[i * W.PU + p] = pick0 ? ((unsigned long long)(i * W.NU + on[0]) << W.PB) | (unsigned long long)p : ~0ull;
      if (cnt > 0 && !pick0) atomicAdd(&W.scal[i * 4 + 2], 1ull);
    }
  }
}

// Round r: one warp per non-empty segment of list buffer r & 1.  k = min(count, m) picks: all m entries when k = m
// (the list empties), else sched_pick_node over the list (k = 1) or over a scratch copy whose entries carry their
// list position (k > 1, where swap-removes reorder the array), each pick tombstoning its list entry.  Pick x of
// segment s owns arrival slot poff[s] + x.
constexpr int WAVE_THREADS = 256;

__global__ void __launch_bounds__(WAVE_THREADS) k_wave_pick(WSched W, int32_t r, long long n_sorted) {
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0 && W.poff[W.nseg] > n_sorted) *W.overflow = 1;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  uint32_t* L = (r & 1) ? W.buf1 : W.buf0;
  for (long long s = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < W.nseg; s += n_warps) {
    const int32_t m = W.len[s];
    if (m == 0) continue;
    const long long i = s / W.NU;
    const long long j = i / W.nc;
    const int32_t c = W.count[i - j * W.nc];
    const int32_t k = m < c ? m : c;
    const long long lo = W.seg_off[s];
    unsigned long long* keys = W.keys_in + W.poff[s];
    uint32_t* Ls = L + lo;
    uint32_t stuck = 0;
    auto take = [&](int32_t x, uint32_t p) {             // the picked partition's cursor advances (the batch completes)
      const long long ci = i * W.PU + p, gp = j * W.PU + p;
      const int cu = W.cur[ci] + 1;
      W.cur[ci] = (uint8_t)cu;
      if (cu >= W.op_n[gp]) { W.part_done[ci] = r + 1; return; }
      const int32_t q2 = W.op_node[gp * W.MO + cu];
      if (wave_pickable(W, q2)) keys[x] = ((unsigned long long)(i * W.NU + q2) << W.PB) | (unsigned long long)p;
      else { W.part_done[ci] = -1; ++stuck; }
    };
    if (k == m) {
      for (int32_t x = lane; x < m; x += 32) take(x, Ls[x] & WAVE_PMASK);
    } else if (k == 1) {                                 // one pick: no swap-remove is ever observed
      sched_pick_node(m, 1, lane, [&](int32_t x) { return Ls[x] >> WAVE_PART_BITS; }, [&](int32_t, int32_t x, int32_t) {
        const uint32_t p = Ls[x] & WAVE_PMASK;
        Ls[x] = p;
        take(0, p);
      });
    } else {
      uint32_t* S = W.scratch + lo;
      for (int32_t x = lane; x < m; x += 32) S[x] = (Ls[x] & ~WAVE_PMASK) | (uint32_t)x;
      __syncwarp();
      sched_pick_node(m, k, lane, [&](int32_t x) { return S[x] >> WAVE_PART_BITS; }, [&](int32_t n, int32_t x, int32_t last) {
        const uint32_t pos = S[x] & WAVE_PMASK;
        const uint32_t p = Ls[pos] & WAVE_PMASK;
        Ls[pos] = p;
        take(n, p);
        S[x] = S[last];
      });
    }
    stuck = __reduce_add_sync(0xFFFFFFFFu, stuck);
    if (lane == 0) {
      if (k == m) W.len[s] = 0;                          // else the merge drops the tombstones
      W.kcnt[s] = 0;                                     // the merge sets it again if the segment is not empty
      W.node_rounds[s] += 1;
      W.node_last[s] = r + 1;
      unsigned long long* sc = W.scal + i * 4;
      sc[0] = (unsigned long long)(r + 1);               // every warp of the instance stores the same value
      atomicAdd(&sc[1], (unsigned long long)k);
      if (stuck) atomicAdd(&sc[2], (unsigned long long)stuck);
      atomicMax(&sc[3], (unsigned long long)k);
    }
  }
}

// [astart, aend) of every segment in the first n sorted keys (padding keys sort last and are ignored).
__global__ void k_wave_bounds(WSched W, long long n) {
  for (long long x = blockIdx.x * (long long)blockDim.x + threadIdx.x; x < n; x += (long long)gridDim.x * blockDim.x) {
    const unsigned long long s = W.keys_out[x] >> W.PB;
    if (s >= (unsigned long long)W.nseg) continue;
    if (x == 0 || (W.keys_out[x - 1] >> W.PB) != s) W.astart[s] = (int32_t)x;
    if (x == n - 1 || (W.keys_out[x + 1] >> W.PB) != s) W.aend[s] = (int32_t)(x + 1);
  }
}

// Round r's merge (r = -1 builds the lists): per touched segment, the survivors of buffer r & 1 in order, merged
// with the segment's arrivals (ascending partition, weights of the ops their cursors now point at) into buffer
// (r + 1) & 1.
__global__ void __launch_bounds__(WAVE_THREADS) k_wave_merge(WSched W, int32_t r) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  const uint32_t* Lin = (r & 1) ? W.buf1 : W.buf0;
  uint32_t* Lout = (r & 1) ? W.buf0 : W.buf1;
  for (long long s = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < W.nseg; s += n_warps) {
    const int32_t m = W.len[s], a0 = W.astart[s], na = W.aend[s] - a0;
    if (m == 0 && na == 0) continue;
    __syncwarp();
    if (lane == 0 && na) { W.astart[s] = 0; W.aend[s] = 0; }
    const long long lo = W.seg_off[s];
    const uint32_t* Ls = Lin + lo;
    uint32_t* Os = Lout + lo;
    uint32_t* S = W.scratch + lo;
    uint32_t* dst = na ? S : Os;
    int32_t ns = 0;
    for (int32_t b = 0; b < m; b += 32) {                // ordered compaction of the survivors
      const uint32_t e = b + lane < m ? Ls[b + lane] : 0u;
      const bool live = (e >> WAVE_PART_BITS) != 0;
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, live);
      if (live) dst[ns + __popc(bal & lt)] = e;
      ns += __popc(bal);
    }
    const long long i = s / W.NU;
    if (na) {
      __syncwarp();
      const unsigned long long* A = W.keys_out + a0;
      const unsigned long long kmask = (1ull << W.PB) - 1;   // a key's partition bits
      const long long j = i / W.nc;
      for (int32_t t = lane; t < ns; t += 32) {
        const uint32_t e = S[t], p = e & WAVE_PMASK;
        int32_t a = 0, b = na;                           // arrivals below p
        while (a < b) { const int32_t h = (a + b) >> 1; if ((uint32_t)(A[h] & kmask) < p) a = h + 1; else b = h; }
        Os[t + a] = e;
      }
      for (int32_t t = lane; t < na; t += 32) {
        const uint32_t p = (uint32_t)(A[t] & kmask);
        int32_t a = 0, b = ns;                           // survivors below p
        while (a < b) { const int32_t h = (a + b) >> 1; if ((S[h] & WAVE_PMASK) < p) a = h + 1; else b = h; }
        const long long gp = j * W.PU + p;
        const uint32_t w = W.op_w[gp * W.MO + W.cur[i * W.PU + p]];
        Os[t + a] = (w << WAVE_PART_BITS) | p;
      }
    }
    if (lane == 0) {
      const int32_t n = ns + na, c = W.count[i - (i / W.nc) * W.nc];
      W.len[s] = n;
      W.kcnt[s] = n < c ? n : c;
    }
  }
}

}  // namespace blance_dev
