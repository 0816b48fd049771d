// blance_b200/csrc/exposure.cuh — the exposure of a rebalance (include/blance_b200.h, blance_moves_exposure and
// blance_plan_scenarios_exposure): the maps M_0 .. M_R a schedule passes through, counted per round without ever
// materialising one of them.  One engine serves a moves handle (one instance, CSR ops, per-op rounds from the
// schedule's order) and a scenario wave (grid y = instance (scenario, count); ops in the wave's fixed-stride table,
// their rounds recorded by k_wave_pick).
//
//   k_expo_op_round   one thread per scheduled op of a handle: op_round[sched_op[i]] = the round whose slice of
//                     sched_op holds i
//   k_expo_walk<0>    one thread per partition: its beg row and ops read once, the per-state entry counts c_s in
//                     registers.  Each state interval [rho_{k-1} + 1, rho_k] contributes its metric values as changes
//                     at the interval's first round into its instance's diff[metric][R + 1] (the t = 0 values
//                     warp-reduced first); the per-partition outputs are written directly, the t = 0 fault-domain
//                     counts with REDs
//   k_expo_series     one CTA per (instance, metric): the scan of diff into the series, its peak, first peak round
//                     and area
//   k_expo_walk<1|2>  (fault domains only) the same walk, counting / emitting (vertex, t, +-1) events where the
//                     partition's deepest common ancestor changes: the chains of the old and the new ancestor below
//                     their own common ancestor.  The events of a group of instances are keyed ((g V + vertex), t)
//                     (g the instance within the group), radix-sorted, merged per key and scanned per key vertex by
//                     the host; k_expo_dom_max takes each vertex's running maximum.
#pragma once

#include <cuda_runtime.h>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "audit.cuh"
#include "blance_b200.h"
#include "device_types.cuh"

namespace blance_dev {

// One instance: a handle's schedule, or one (scenario, count) pair of a wave.
struct ExpoInst {
  long long beg_off;              // its beg rows: beg + beg_off + p * stride
  long long pf_off;               // its partitions' begMap flags: pflags + pf_off + p
  long long gp_off;               // its partitions' ops: partition gp_off + p of the op source
  long long diff_off;             // its [BLANCE_EXPO_N][R + 1] slice of diff
  int32_t R;
  int32_t constraints[BL_S_MAX];
};

struct ExpoArgs {
  const ExpoInst* inst;           // [ni]
  const long long* op_off;        // [P + 1] CSR ops of a handle (one instance), or NULL: the table [.][MO], op_n
  const uint8_t* op_n;
  const int32_t* op_node;
  const uint8_t* op_state;
  const uint8_t* op_kind;
  const int32_t* op_round;        // round of each op, -1 = never scheduled: CSR [total_ops] / table [ni * P][MO]
  const int32_t* beg;             // beg rows, `stride` apart
  const uint8_t* pflags;          // begMap membership (PF_IN_PREV | PF_IN_ASSIGN), or NULL: every partition, its row
  const int32_t* dom_parent;      // [V] or NULL (every node its own root)
  long long* diff;                // the instances' [BLANCE_EXPO_N][R + 1] changes, scanned in place into the series
  int32_t* part_min;              // [ni][P] or NULL
  int32_t* part_notop;            // [ni][P] or NULL
  uint8_t* part_flags;            // [ni][P] or NULL
  long long* dom_base;            // [ni][V] partitions under each vertex in M_0, or NULL (no fault domains asked for)
  long long* ev_count;            // [ni * P + 1] events per (instance, partition) (pass 1)
  const long long* ev_off;        // [ni * P + 1] their exclusive scan (pass 2), ev0 = that of the group's first
  unsigned long long* ev_key;     // ((g V + vertex) << 32) | t, g = instance - g0
  int32_t* ev_val;                // +1 / -1
  long long stride, ev0;
  int32_t P, SL, S, NU, V, MO, top;
  int32_t i0;                     // the launch's first instance (grid y is at most 65535 instances)
  int32_t g0;                     // the first instance of the event group being emitted (pass 2)
  int32_t slot_off[BL_S_MAX + 1];
};

// the metric values of one partition with entry counts c[] under constraints cons[BL_S_MAX] (enum
// blance_expo_metric order)
__device__ __forceinline__ void expo_values(const ExpoArgs& E, const int32_t* cons, const int (&c)[BL_S_MAX], int (&v)[BLANCE_EXPO_N]) {
  int C = 0, ctop = 0, ktop = 0;
  bool is_short = false;
#pragma unroll
  for (int s = 0; s < BL_S_MAX; ++s) {                // c[s] = 0 for s >= S
    C += c[s];
    const int at_top = -(int)(s == E.top);          // masks, not selects: a select folds into c[top], a local-memory load
    ctop += c[s] & at_top;
    ktop += cons[s] & at_top;
    is_short |= s < E.S && cons[s] > 0 && c[s] < cons[s];
  }
  const bool has_top = E.top >= 0;
  v[BLANCE_EXPO_NO_TOP] = has_top && ctop == 0;
  v[BLANCE_EXPO_MULTI_TOP] = has_top && ktop > 0 && ctop > ktop;
  v[BLANCE_EXPO_SHORT] = is_short;
  v[BLANCE_EXPO_ONE_COPY] = C == 1;
  v[BLANCE_EXPO_NO_COPY] = C == 0;
  v[BLANCE_EXPO_COPIES] = C;
}

// the state that owns slot i
__device__ __forceinline__ int expo_slot_state(const ExpoArgs& E, int i) {
  int si = 0;
#pragma unroll
  for (int s = 1; s < BL_S_MAX; ++s) si += (s < E.S && i >= E.slot_off[s]) ? 1 : 0;
  return si;
}

// one more entry on node x folded into a deepest common ancestor d (-2: no entry yet, -1: under no vertex)
__device__ __forceinline__ int expo_fold(const ExpoArgs& E, int d, int32_t x) {
  if (x < 0 || x >= E.NU) return -1;
  return d == -2 ? x : d == -1 ? -1 : audit_dca(E.dom_parent, d, x);
}

// The deepest common ancestor of a partition's entries after its first n_applied ops: the beg entries whose node has
// not had its op yet, and the node of every applied op that is not a del.  -1 when there is none.
__device__ __forceinline__ int expo_dca(const ExpoArgs& E, const int32_t* row, uint32_t live, long long o0, long long n_applied) {
  int d = -2;
  for (uint32_t m = live; m; m &= m - 1) d = expo_fold(E, d, row[__ffs(m) - 1]);
  for (long long k = o0; k < o0 + n_applied; ++k)
    if (E.op_kind[k] != BLANCE_OP_DEL) d = expo_fold(E, d, E.op_node[k]);
  return d < 0 ? -1 : d;
}

// Calls f(v) for the vertices from d up to, not including, stop (-1: up to the root).
template <class F>
__device__ __forceinline__ void expo_chain(const ExpoArgs& E, int d, int stop, F&& f) {
  for (int v = d, i = 0; v >= 0 && v != stop && i <= AUDIT_DEPTH_MAX; v = audit_parent(E.dom_parent, v), ++i) f(v);
}

__global__ void k_expo_op_round(long long moves_done, int32_t R, const long long* __restrict__ round_off,
                                const long long* __restrict__ sched_op, int32_t* __restrict__ op_round) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < moves_done; i += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = R - 1;                        // the round r with round_off[r] <= i < round_off[r + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (round_off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    op_round[sched_op[i]] = lo;
  }
}

// MODE 0: metrics, per-partition outputs and the t = 0 domain counts; 1: count domain events; 2: emit them.
// Grid: x strides over the partitions of instance i0 + blockIdx.y.
template <int MODE>
__global__ void __launch_bounds__(256) k_expo_walk(const ExpoArgs E) {
  __shared__ ExpoInst I;
  const int i = E.i0 + blockIdx.y;
  if (threadIdx.x == 0) I = E.inst[i];
  __syncthreads();
  const long long R1 = (long long)I.R + 1;
  long long* diff = E.diff + I.diff_off;
  // warp-uniform trip count: every lane reaches the t = 0 reductions at the end of each pass
  for (long long p0 = blockIdx.x * (long long)blockDim.x; p0 < E.P; p0 += (long long)gridDim.x * blockDim.x) {
    const long long p = p0 + threadIdx.x, ci = (long long)i * E.P + p;
    uint32_t base[BLANCE_EXPO_N] = {0, 0, 0, 0, 0, 0};
    const uint8_t f = p < E.P && E.pflags ? E.pflags[I.pf_off + p] : (uint8_t)PF_IN_PREV;
    if (p < E.P && !(f & (PF_IN_PREV | PF_IN_ASSIGN))) {     // in neither map: no partition of begMap
      if (MODE == 0) {
        if (E.part_min) E.part_min[ci] = -1;
        if (E.part_notop) E.part_notop[ci] = 0;
        if (E.part_flags) E.part_flags[ci] = 0;
      }
      if (MODE == 1) E.ev_count[ci] = 0;
    } else if (p < E.P) {
      const int32_t* row = E.beg + I.beg_off + p * E.stride;
      const long long gp = I.gp_off + p;
      const long long o0 = E.op_off ? E.op_off[gp] : gp * E.MO;
      const long long o1 = E.op_off ? E.op_off[gp + 1] : o0 + E.op_n[gp];
      const int32_t* rho = E.op_round + (E.op_off ? 0 : ci * E.MO - o0);
      int c[BL_S_MAX] = {0, 0, 0, 0, 0, 0, 0, 0};
      uint32_t live = 0, closed = 0;                 // beg slots that hold an entry whose node has not had its op yet;
      for (int x = 0; x < E.SL && (f & PF_IN_PREV); ++x) {   // states whose list already ended (no row: empty)
        const int si = expo_slot_state(E, x);
        if (row[x] == BLANCE_NO_NODE || (closed >> si & 1u)) { closed |= 1u << si; continue; }
        live |= 1u << x;
#pragma unroll
        for (int s = 0; s < BL_S_MAX; ++s) c[s] += s == si ? 1 : 0;
      }
      int v[BLANCE_EXPO_N];
      expo_values(E, I.constraints, c, v);
      int min_c = v[BLANCE_EXPO_COPIES], notop = 0, t0 = 0;
      uint32_t flags = 0;
      if (MODE == 0) {
#pragma unroll
        for (int m = 0; m < BLANCE_EXPO_N; ++m) { base[m] += (uint32_t)v[m]; flags |= (v[m] != 0) << m; }
        if (E.dom_base) {
          const int d = expo_dca(E, row, live, o0, 0);
          expo_chain(E, d, -1, [&](int x) { red_add64(E.dom_base + (long long)i * E.V + x, 1ull); });
        }
      }
      int d_prev = MODE == 0 ? -1 : expo_dca(E, row, live, o0, 0);
      long long n_ev = 0, w = MODE == 2 ? E.ev_off[ci] - E.ev0 : 0;
      for (long long k = o0; k < o1; ++k) {
        const int r = rho[k];
        if (r < 0) break;                            // the partition is stuck from here on
        // apply op k: every entry of its node leaves, a non-del op adds one entry of its state (one op per node, so
        // the entries that leave are exactly the node's beg entries)
        const int32_t n = E.op_node[k];
        for (uint32_t m = live; m; m &= m - 1) {
          const int x = __ffs(m) - 1;
          if (row[x] != n) continue;
          live &= ~(1u << x);
          const int si = expo_slot_state(E, x);
#pragma unroll
          for (int s = 0; s < BL_S_MAX; ++s) c[s] -= s == si ? 1 : 0;
        }
        const uint8_t kind = E.op_kind[k], st = E.op_state[k];
        if (kind != BLANCE_OP_DEL) {
#pragma unroll
          for (int s = 0; s < BL_S_MAX; ++s) c[s] += s == st ? 1 : 0;
        }
        if (MODE == 0) {
          notop += v[BLANCE_EXPO_NO_TOP] * (r + 1 - t0);       // the state before held rounds t0 .. r
          int u[BLANCE_EXPO_N];
          expo_values(E, I.constraints, c, u);
#pragma unroll
          for (int m = 0; m < BLANCE_EXPO_N; ++m) {
            if (u[m] != v[m]) red_add64(diff + m * R1 + r + 1, (unsigned long long)(long long)(u[m] - v[m]));
            flags |= (u[m] != 0) << m;
            v[m] = u[m];
          }
          min_c = min(min_c, v[BLANCE_EXPO_COPIES]);
        } else {
          const int d = expo_dca(E, row, live, o0, k - o0 + 1);
          if (d != d_prev) {
            const int top = d_prev >= 0 && d >= 0 ? audit_dca(E.dom_parent, d_prev, d) : -1;
            const unsigned long long t = (unsigned long long)(r + 1);
            const unsigned long long g = (unsigned long long)(i - E.g0) * (unsigned long long)E.V;
            auto ev = [&](int x, int32_t delta) {
              if (MODE == 2) { E.ev_key[w] = ((g + (unsigned long long)x) << 32) | t; E.ev_val[w] = delta; ++w; }
              else ++n_ev;
            };
            expo_chain(E, d_prev, top, [&](int x) { ev(x, -1); });
            expo_chain(E, d, top, [&](int x) { ev(x, 1); });
            d_prev = d;
          }
        }
        t0 = r + 1;
      }
      if (MODE == 0) {
        notop += v[BLANCE_EXPO_NO_TOP] * (I.R + 1 - t0);
        if (E.part_min) E.part_min[ci] = min_c;
        if (E.part_notop) E.part_notop[ci] = notop;
        if (E.part_flags) E.part_flags[ci] = (uint8_t)flags;
      }
      if (MODE == 1) E.ev_count[ci] = n_ev;
    }
    if (MODE == 0) {
      // every partition's t = 0 values land on index 0: one RED per warp and metric
#pragma unroll
      for (int m = 0; m < BLANCE_EXPO_N; ++m) {
        const uint32_t b = __reduce_add_sync(0xFFFFFFFFu, base[m]);
        if ((threadIdx.x & 31) == 0 && b) red_add64(diff + m * R1, b);
      }
    }
  }
}

// One CTA per (metric blockIdx.x, instance blockIdx.y): the instance's diff[m] scanned in place into series[m];
// stats[instance][m] = {peak, first round at the peak, area}.
__global__ void __launch_bounds__(512) k_expo_series(const ExpoInst* __restrict__ inst, long long* __restrict__ diff,
                                                     long long* __restrict__ stats) {
  typedef cub::BlockScan<long long, 512> Scan;
  typedef cub::BlockReduce<long long, 512> Reduce;
  __shared__ typename Scan::TempStorage s_scan;
  __shared__ typename Reduce::TempStorage s_red;
  __shared__ long long s_carry, s_peak;
  const ExpoInst& I = inst[blockIdx.y];
  const long long n = (long long)I.R + 1;
  long long* x = diff + I.diff_off + blockIdx.x * n;
  stats += ((long long)blockIdx.y * BLANCE_EXPO_N + blockIdx.x) * 3;
  long long best = LLONG_MIN, best_t = LLONG_MAX, area = 0;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (long long b = 0; b < n; b += blockDim.x) {
    const long long i = b + threadIdx.x;
    long long val = i < n ? x[i] : 0, total;
    Scan(s_scan).InclusiveSum(val, val, total);
    val += s_carry;
    __syncthreads();                               // every thread has read the carry
    if (threadIdx.x == 0) s_carry += total;
    if (i < n) {
      x[i] = val;
      area += val;
      if (val > best) { best = val; best_t = i; }  // i ascends per thread: the first index at this thread's max
    }
    __syncthreads();
  }
  const long long peak = Reduce(s_red).Reduce(best, [](long long a, long long b) { return a > b ? a : b; });
  if (threadIdx.x == 0) s_peak = peak;
  __syncthreads();
  const long long first = Reduce(s_red).Reduce(best == s_peak ? best_t : LLONG_MAX, [](long long a, long long b) { return a < b ? a : b; });
  __syncthreads();
  const long long sum = Reduce(s_red).Sum(area);
  if (threadIdx.x == 0) {
    stats[0] = s_peak; stats[1] = first; stats[2] = sum;
  }
}

// the merge of events with one (vertex, t) key and the running sum of one vertex's merged events
struct ExpoSum {
  __host__ __device__ int32_t operator()(int32_t a, int32_t b) const { return a + b; }
};
struct ExpoSameVertex {
  __host__ __device__ bool operator()(unsigned long long a, unsigned long long b) const { return (a >> 32) == (b >> 32); }
};

// dom_key[v] = (partitions under v << 32) | (0xFFFFFFFF - t) at t = 0, over the n = instances x V vertices: the running
// maximum starts there.
__global__ void k_expo_dom_init(long long n, const long long* __restrict__ dom_base, unsigned long long* __restrict__ dom_key) {
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x)
    dom_key[v] = ((unsigned long long)dom_base[v] << 32) | 0xFFFFFFFFu;
}

// Run i of the merged events: (key vertex, t) and the key vertex's running sum of changes up to and including t.  The
// count at t is dom_base + that sum; the largest count, at its smallest t, wins the RED.MAX on one u64 key.  A key
// vertex g V + v is vertex v of the group's instance g: dom_base and dom_key are the group's [g][V] slices.
__global__ void k_expo_dom_max(int n, const unsigned long long* __restrict__ keys,
                               const int32_t* __restrict__ running, const long long* __restrict__ dom_base,
                               unsigned long long* __restrict__ dom_key) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long key = keys[i];
    const long long v = (long long)(key >> 32);
    const uint32_t t = (uint32_t)key;
    const unsigned long long cnt = (unsigned long long)(dom_base[v] + running[i]);
    red_max64((long long*)(dom_key + v), (cnt << 32) | (0xFFFFFFFFu - t));
  }
}

// The span of a chain wave (blance_plan_chains_exposure): one stage's schedule summaries, per-partition exposures and
// fault-domain maxima folded into per-instance accumulators.  Inputs are [ni][NU], [ni][PU] and [ni][V] as the
// schedule (WSched), the exposure walk (ExpoArgs) and k_expo_dom_max leave them; a null input or accumulator is not
// folded.  G[i] is the global round at which this stage starts for instance i.
struct ChainFold {
  const int32_t* node_rounds; const int32_t* node_last; const int32_t* part_done;
  const int32_t* part_min; const int32_t* part_notop; const uint8_t* part_flags;
  const unsigned long long* dom_key;
  const long long* G;
  int32_t* a_node_rounds; long long* a_node_last; long long* a_part_done;
  int32_t* a_part_min; int32_t* a_part_notop; uint8_t* a_part_flags;
  long long* a_dom_peak; int32_t* a_dom_stage; int32_t* a_dom_round;
  long long ni;
  int32_t PU, NU, V, stage;
};

// One thread per accumulator element (instance, partition | node | vertex), stages folded in launch order: no atomics.
// Stage 0 starts every accumulator from its identity instead of reading it.
__global__ void __launch_bounds__(256) k_chain_fold(const ChainFold F) {
  const long long W = (long long)F.PU + F.NU + F.V, n = F.ni * W;
  const bool first = F.stage == 0;
  for (long long x = blockIdx.x * (long long)blockDim.x + threadIdx.x; x < n; x += (long long)gridDim.x * blockDim.x) {
    const long long i = x / W, e = x - i * W, G = F.G[i];
    if (e < F.PU) {
      const long long c = i * F.PU + e;
      if (F.a_part_done) {
        const long long old = first ? 0 : F.a_part_done[c];
        const int32_t d = F.part_done[c];
        F.a_part_done[c] = old == -1 || d == -1 ? -1 : d > 0 ? G + d : old;
      }
      if (F.a_part_min) {
        const int32_t old = first ? -1 : F.a_part_min[c], m = F.part_min[c];
        F.a_part_min[c] = m < 0 ? old : old < 0 ? m : min(old, m);
      }
      if (F.a_part_notop) F.a_part_notop[c] = (first ? 0 : F.a_part_notop[c]) + F.part_notop[c];
      if (F.a_part_flags) F.a_part_flags[c] = (uint8_t)((first ? 0 : F.a_part_flags[c]) | F.part_flags[c]);
    } else if (e < F.PU + F.NU) {
      const long long c = i * F.NU + (e - F.PU);
      if (F.a_node_rounds) F.a_node_rounds[c] = (first ? 0 : F.a_node_rounds[c]) + F.node_rounds[c];
      if (F.a_node_last) {
        const int32_t l = F.node_last[c];
        F.a_node_last[c] = l > 0 ? G + l : first ? 0 : F.a_node_last[c];
      }
    } else if (F.a_dom_peak) {
      const long long c = i * F.V + (e - F.PU - F.NU);
      const unsigned long long key = F.dom_key[c];
      const long long cnt = (long long)(key >> 32);
      if (first || cnt > F.a_dom_peak[c]) {
        F.a_dom_peak[c] = cnt;
        F.a_dom_stage[c] = F.stage;
        F.a_dom_round[c] = (int32_t)(0xFFFFFFFFu - (uint32_t)key);
      }
    }
  }
}

}  // namespace blance_dev
