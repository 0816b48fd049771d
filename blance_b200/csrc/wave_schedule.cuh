// blance_b200/csrc/wave_schedule.cuh — the lock-step schedule of include/blance_b200.h (blance_moves_schedule):
// rounds of findAvailableMovesUnlocked (orchestrate.go:749-763) followed, per node, by
// filterNextPlausibleMovesForNode (orchestrate.go:482-504) with LowestWeightPartitionMoveForNode
// (orchestrate.go:177-186).  One engine computes it for a moves handle (blance_moves_schedule: one instance, with
// the per-op order) and for every scenario of a blance_plan_scenarios_schedule wave at once (reduced to per-node
// and per-partition summaries).
//
// An instance is a pair (scenario j of the wave, count index k): i = j * nc + k.  All instances run in lock step:
// global round r is round r of every instance that still has entries.  A segment is one (instance, node q) pair,
// s = i * NU + q.  The engine keeps, per segment, the list findAvailableMovesUnlocked builds: the partitions whose
// next op is on q, in ascending partition index, each entry (MoveOpWeight << 29) | p.  A partition has at most one
// op per node (CalcPartitionMoves' "seen" rule), so a segment never holds more entries than its scenario has ops on
// its node: the host carves segment capacities from those counts.
//
// Between rounds a list changes only by its own picks leaving and by partitions arriving from picks elsewhere, so
// a round is a fixed launch sequence whose work follows the list entries and the round's picks:
//   scan           of the segments' pick counts min(count, length): each segment's slots for its arrival keys
//   k_wave_pick    one warp per non-empty segment: sched_pick_node, picked entries tombstoned (weight bits 0) in
//                  place, summaries and cursors updated, and the arrival key (segment of the next op << PB) | p
//                  written for every picked partition with a pickable next op
//   radix sort     of the round's arrival slots only (a host bound on the picks, padded with ~0)
//   k_wave_bounds  the slice of the sorted arrivals of each segment that received any
//   k_wave_merge   one warp per touched segment: survivors (in order) merged with its arrivals into the other list
//                  buffer, and its next pick count
// The lists are first built by the same sort, bounds and merge from the keys k_wave_first writes for every
// partition's first op.  A round without picks changes nothing, so the host enqueues blocks of rounds and reads the
// last round's pick count once per block.
//
// The ops are a moves handle's CSR arrays (op_off set) or the table [nw * PU][MO] k_wave_moves fills.  With one
// instance the segments are the nodes in ascending id, so pick x of segment s in round r is op
// round_off[r] + poff[s] + x of the schedule's order (round, node id, pick order).  For an exposure of the table's
// schedules (exposure.cuh), k_wave_moves also keeps each op's state and k_wave_pick each op's round per instance.
#pragma once

#include <cuda_runtime.h>

#include "aux_kernels.cuh"
#include "blance_b200.h"

namespace blance_dev {

constexpr int WAVE_PART_BITS = 29;                          // entry = (weight << 29) | partition; weight 0 = picked
constexpr uint32_t WAVE_PMASK = (1u << WAVE_PART_BITS) - 1;

struct WSched {
  int32_t nw, nc, PU, NU, MO, PB;          // scenarios, counts, partitions per scenario, node ids, ops per partition, key bits of p
  long long nseg;                          // nw * nc * NU
  const int32_t* count;                    // [nc] picks per node and round (max(1, MaxConcurrentPartitionMovesPerNode))
  const uint8_t* mover;                    // [NU]
  const long long* op_off;                 // [nw * PU + 1] CSR offsets of the ops, or null: the op table
  uint8_t* op_n;                           // [nw * PU] ops per partition of the op table
  int32_t* op_node; uint8_t* op_kind;      // the ops: CSR [op_off[nw * PU]] or table [nw * PU][MO]
  int32_t* cur; int32_t* part_done;        // [ni * PU]: cursor, part_done_round
  const long long* seg_off;                // [nseg + 1] segment capacities
  int32_t* len; int32_t* kcnt;             // [nseg + 1]: list length, picks of the next round (kcnt[nseg] = 0)
  const long long* poff;                   // [nseg + 1] exclusive scan of kcnt: arrival slots, poff[nseg] = picks
  int32_t* astart; int32_t* aend; int32_t* node_rounds; int32_t* node_last;   // [nseg]
  uint32_t* buf0; uint32_t* buf1; uint32_t* scratch;                          // [seg_off[nseg]]
  unsigned long long* keys_in; const unsigned long long* keys_out;             // arrival keys
  unsigned long long* scal;                // [ni][4]: rounds, moves_done, stuck_parts, max_batch
  int32_t* overflow;                       // more picks than the host sorted (internal error)
  long long* esum;                         // the host's reduction of len: entries left in all lists
  long long* round_off; long long* sched_op;   // one instance only: the per-op order (null: not emitted)
  uint8_t* op_state;                       // [nw * PU][MO] the op table's states, or null (no exposure asked for)
  int32_t* op_round;                       // [ni * PU][MO] the round of each op of the table, -1 = never; or null
};

__device__ __forceinline__ bool wave_pickable(const WSched& W, int32_t node) {
  return node >= 0 && node < W.NU && W.mover[node] != 0;
}

// index of op c of partition gp (= j * PU + p) in op_node / op_kind, and gp's op count
__device__ __forceinline__ long long wave_op(const WSched& W, long long gp, int32_t c) {
  return W.op_off ? W.op_off[gp] + c : gp * W.MO + c;
}

__device__ __forceinline__ int32_t wave_n_ops(const WSched& W, long long gp) {
  return W.op_off ? (int32_t)(W.op_off[gp + 1] - W.op_off[gp]) : W.op_n[gp];
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

// ops per node id in [0, NU) of the n CSR ops of a moves handle: its segment capacities
__global__ void k_wave_node_ops(long long n, const int32_t* __restrict__ op_node, int32_t NU, unsigned long long* __restrict__ cnt) {
  for (long long x = blockIdx.x * (long long)blockDim.x + threadIdx.x; x < n; x += (long long)gridDim.x * blockDim.x) {
    const int32_t q = op_node[x];
    if (q >= 0 && q < NU) atomicAdd(&cnt[q], 1ull);
  }
}

// CalcPartitionMoves of every assigned partition of every scenario into the op table (the rules of
// k_scenario_summary: the prev row as uploaded, an empty row for a partition absent from prevMap).  Grid: x strides
// over the partitions of scenario blockIdx.y.
__global__ void k_wave_moves(DPool pool, const int32_t* __restrict__ prev_rows_init, const uint8_t* __restrict__ pflags_init,
                             int32_t favor_min, WSched W) {
  const int j = blockIdx.y;
  const DInst& D = pool.insts[j];
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < D.PU; p += (long long)gridDim.x * blockDim.x) {
    const long long g = D.part_off + p;
    const long long gp = (long long)j * W.PU + p;
    const uint8_t f = pflags_init[g];
    int32_t* on = W.op_node + gp * W.MO;
    uint8_t* ok = W.op_kind + gp * W.MO;
    uint8_t* os = W.op_state ? W.op_state + gp * W.MO : nullptr;
    int cnt = 0;
    if (f & PF_IN_ASSIGN) {
      auto emit = [&](int32_t node, int state, int kind) {
        for (int x = 0; x < cnt; ++x) if (on[x] == node) return;   // addMoves + seen, moves.go:51-58
        on[cnt] = node; ok[cnt] = (uint8_t)kind;
        if (os) os[cnt] = (uint8_t)state;
        ++cnt;
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
  }
}

// Per instance, every partition's cursor and done round, and its first op: its arrival key in slot i * PU + p when
// the op's node has a mover, else the partition is stuck.  Grid: x strides over the partitions of scenario blockIdx.y.
__global__ void k_wave_first(WSched W) {
  const int j = blockIdx.y;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < W.PU; p += (long long)gridDim.x * blockDim.x) {
    const long long gp = (long long)j * W.PU + p;
    const int32_t n = wave_n_ops(W, gp);
    const int32_t q = n > 0 ? W.op_node[wave_op(W, gp, 0)] : -1;
    const bool pick0 = n > 0 && wave_pickable(W, q);
    for (int k = 0; k < W.nc; ++k) {
      const long long i = (long long)j * W.nc + k;
      W.cur[i * W.PU + p] = 0;
      W.part_done[i * W.PU + p] = n == 0 || pick0 ? 0 : -1;
      W.keys_in[i * W.PU + p] = pick0 ? ((unsigned long long)(i * W.NU + q) << W.PB) | (unsigned long long)p : ~0ull;
      if (n > 0 && !pick0) atomicAdd(&W.scal[i * 4 + 2], 1ull);
    }
  }
}

// Round r: one warp per non-empty segment of list buffer r & 1.  k = min(count, m) picks: all m entries in list
// order when k = m (the list empties) and that order is not an output, else sched_pick_node over the list (k = 1)
// or over a scratch copy whose entries carry their list position (k > 1, where swap-removes reorder the array),
// each pick tombstoning its list entry and parking its partition in its arrival slot until the warp takes the
// picks in parallel.  Pick x of segment s owns arrival slot poff[s] + x (~0 when the partition does not arrive
// anywhere); the slots past the round's picks up to the host's sort bound are padded with ~0.  A round with picks
// advances round_off.
constexpr int WAVE_THREADS = 256;

__global__ void __launch_bounds__(WAVE_THREADS) k_wave_pick(WSched W, int32_t r, long long n_sorted) {
  const int lane = threadIdx.x & 31;
  const long long picks = W.poff[W.nseg];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (picks > n_sorted) *W.overflow = 1;
    if (W.round_off && picks > 0) W.round_off[r + 1] = W.round_off[r] + picks;
  }
  for (long long x = picks + blockIdx.x * (long long)blockDim.x + threadIdx.x; x < n_sorted; x += (long long)gridDim.x * blockDim.x)
    W.keys_in[x] = ~0ull;                                // the sort's padding past the round's picks
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
    long long* ops = W.sched_op ? W.sched_op + W.round_off[r] + W.poff[s] : nullptr;
    uint32_t* Ls = L + lo;
    uint32_t stuck = 0;
    auto take = [&](int32_t x, uint32_t p) {             // the picked partition's cursor advances (the batch completes)
      const long long ci = i * W.PU + p, gp = j * W.PU + p;
      const int32_t cu = W.cur[ci];
      if (ops) ops[x] = wave_op(W, gp, cu);
      if (W.op_round) W.op_round[ci * W.MO + cu] = r;
      W.cur[ci] = cu + 1;
      unsigned long long key = ~0ull;
      if (cu + 1 >= wave_n_ops(W, gp)) W.part_done[ci] = r + 1;
      else {
        const int32_t q2 = W.op_node[wave_op(W, gp, cu + 1)];
        if (wave_pickable(W, q2)) key = ((unsigned long long)(i * W.NU + q2) << W.PB) | (unsigned long long)p;
        else { W.part_done[ci] = -1; ++stuck; }
      }
      keys[x] = key;
    };
    if (k == m && (m == 1 || !ops)) {
      for (int32_t x = lane; x < m; x += 32) take(x, Ls[x] & WAVE_PMASK);
    } else {
      if (k == 1) {                                      // one pick: no swap-remove is ever observed
        sched_pick_node(m, 1, lane, [&](int32_t x) { return Ls[x] >> WAVE_PART_BITS; }, [&](int32_t, int32_t x, int32_t) {
          const uint32_t p = Ls[x] & WAVE_PMASK;
          Ls[x] = p;
          keys[0] = p;
        });
      } else {
        uint32_t* S = W.scratch + lo;
        for (int32_t x = lane; x < m; x += 32) S[x] = (Ls[x] & ~WAVE_PMASK) | (uint32_t)x;
        __syncwarp();
        sched_pick_node(m, k, lane, [&](int32_t x) { return S[x] >> WAVE_PART_BITS; }, [&](int32_t n, int32_t x, int32_t last) {
          const uint32_t pos = S[x] & WAVE_PMASK;
          const uint32_t p = Ls[pos] & WAVE_PMASK;
          Ls[pos] = p;
          keys[n] = p;
          S[x] = S[last];
        });
      }
      __syncwarp();
      for (int32_t x = lane; x < k; x += 32) take(x, (uint32_t)keys[x]);
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
        const uint32_t w = (uint32_t)move_op_weight(W.op_kind[wave_op(W, gp, W.cur[i * W.PU + p])]);
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
