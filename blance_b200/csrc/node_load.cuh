// blance_b200/csrc/node_load.cuh — each node's load over the maps a rebalance passes through (blance_moves_load,
// include/blance_b200.h); c_abi.cu launches them (load_run).
//
//   k_load_walk<0>   one thread per partition: its beg entries' weights RED into node_beg (lanes that share a
//                    (state, node) index merged first), and the number of events its scheduled ops emit
//   k_load_walk<1>   the same walk, emitting the events at the partition's exclusive offset: an op on node n applied
//                    at round rho + 1 takes away n's beg entries and, unless it is a del, adds one entry (n, s_op);
//                    each nonzero change of (n, s) and the net change of (n, S) is one event
//                    ((n (S + 1) + s) << 32 | rho + 1, change).  The seen rule (moves.go:51-58) gives n at most one
//                    op per partition, so its entries before that op are exactly its beg entries.
//   k_load_init      peak_key = pack(node_beg, 0) (the load at t = 0) and node_end = node_beg
//   k_load_peak      one thread per merged (key, t) run after the per-key inclusive scan: the load at t is node_beg
//                    plus the running sum; one RED.MAX.64 of pack(load, t) per run, and the key's last run writes
//                    node_end
//   k_load_final     node_peak / node_peak_round from peak_key, and one RED.MAX.64 per warp of
//                    (overshoot << 32) | ~q over the nodes' all-state rows
// |load| stays below 2^31 (the host's count bound; a wave's partition weights may be negative, as the planner allows),
// so every change, merged run and running sum fits an int32, and pack(load, t) = ((load + 2^31) << 32) | ~t orders
// loads, then earlier rounds, as unsigned 64-bit keys: the packed maxima are exact.
#pragma once

#include <cuda_runtime.h>

#include "blance_b200.h"
#include "device_types.cuh"

namespace blance_load {

struct LoadArgs {
  // one instance: a moves handle's beg rows and CSR ops, or one (scenario, count) of a wave with its ops in a table
  // of MO per partition; the round of each op (-1 = never scheduled) is laid out as the ops are
  const int32_t* beg;               // [P] rows, `stride` apart
  const long long* op_off;          // [P + 1] CSR, or NULL: partition p's ops are [p MO, p MO + op_n[p])
  const uint8_t* op_n;              // [P] (table form)
  const int32_t* op_node;
  const uint8_t* op_state;
  const uint8_t* op_kind;
  const int32_t* op_round;
  const int32_t* weight;            // [P], or NULL: every partition weighs 1
  const uint8_t* pflags;            // [P] begMap membership (PF_IN_PREV | PF_IN_ASSIGN) and PF_HAS_WEIGHT, or NULL: every
                                    // partition has its row and, with `weight`, its weight
  int32_t has_part_weights;         // with pflags: weight[p] applies where pflags[p] has PF_HAS_WEIGHT
  long long stride;
  int32_t P, S, SL, NU, MO;
  int32_t slot_off[9];              // [S + 1]
  // results, [S + 1][NU] each (row S: every state)
  long long* node_beg;
  long long* node_end;
  long long* node_peak;
  int32_t* node_peak_round;
  unsigned long long* peak_key;     // ((load + 2^31) << 32) | ~t, the running maximum
  unsigned long long* over_key;     // [1] (overshoot << 32) | ~q
  // the event count per partition and its exclusive scan, [P + 1] each
  long long* ev_count;
  long long* ev_off;
  void* scan_tmp;
  size_t scan_tmp_bytes;
  // the events, [NE] each, and the sort / merge / scan scratch
  unsigned long long *ev_key, *ev_key2, *run_key;
  int32_t *ev_val, *ev_val2, *run_val, *run_sum;
  int* n_runs;
  void* ev_tmp;
  size_t ev_tmp_bytes;
};

// reductions nobody waits for: red.* in global memory, never an atomic whose result is thrown away
__device__ __forceinline__ void red_add64(long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_max64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// Adds w at index key (-1: nowhere) for every lane of the warp: lanes with the same key are summed first and their
// lowest lane issues the one RED.  Every lane calls it.  The sum of one index fits 32 bits: it is part of a load.
__device__ __forceinline__ void red_merged(long long* base, long long key, int32_t w) {
  const unsigned grp = __match_any_sync(0xFFFFFFFFu, key);
  const int32_t sum = __reduce_add_sync(grp, w);
  if (key >= 0 && sum && (int)(threadIdx.x & 31) == __ffs(grp) - 1) red_add64(base + key, (unsigned long long)(long long)sum);
}

__device__ __forceinline__ unsigned long long pack(long long load, uint32_t t) {
  return ((unsigned long long)(load + (1ll << 31)) << 32) | (0xFFFFFFFFu - t);
}

__device__ __forceinline__ int slot_state(const LoadArgs& A, int x) {
  int si = 0;
#pragma unroll
  for (int s = 1; s < BL_S_MAX; ++s) si += (s < A.S && x >= A.slot_off[s]) ? 1 : 0;
  return si;
}

template <int MODE>
__global__ void __launch_bounds__(256) k_load_walk(const LoadArgs A) {
  const long long NU = A.NU;
  // warp-uniform trip count: every lane reaches the merged REDs
  for (long long p0 = blockIdx.x * (long long)blockDim.x; p0 < A.P; p0 += (long long)gridDim.x * blockDim.x) {
    const long long p = p0 + threadIdx.x;
    const bool in = p < A.P;
    const int32_t* row = A.beg + (in ? p : 0) * A.stride;
    const uint8_t f = in && A.pflags ? A.pflags[p] : (uint8_t)PF_IN_PREV;
    const bool part = in && (f & (PF_IN_PREV | PF_IN_ASSIGN));   // a partition of begMap
    const int32_t w = in && A.weight && (!A.pflags || (A.has_part_weights && (f & PF_HAS_WEIGHT))) ? A.weight[p] : 1;
    uint32_t live = 0, closed = 0;                 // beg slots with an entry whose node has not had its op yet;
    for (int x = 0; x < A.SL && in && (f & PF_IN_PREV); ++x) {   // states whose list already ended (no row: empty)
      const int si = slot_state(A, x);
      if (row[x] == BLANCE_NO_NODE || (closed >> si & 1u)) { closed |= 1u << si; continue; }
      live |= 1u << x;
    }
    if (MODE == 0) {
      for (int x = 0; x < A.SL; ++x) {
        const int32_t n = (live >> x & 1u) ? row[x] : -1;
        const bool ok = n >= 0 && n < A.NU;
        red_merged(A.node_beg, ok ? slot_state(A, x) * NU + n : -1, w);
        red_merged(A.node_beg, ok ? A.S * NU + n : -1, w);
      }
    }
    if (!part) {
      if (MODE == 0 && in) A.ev_count[p] = 0;
      continue;
    }
    long long n_ev = 0, at = MODE == 1 ? A.ev_off[p] : 0;
    const long long o0 = A.op_off ? A.op_off[p] : p * A.MO, o1 = A.op_off ? A.op_off[p + 1] : o0 + A.op_n[p];
    for (long long k = o0; k < o1; ++k) {
      const int r = A.op_round[k];
      if (r < 0) break;                            // the partition is stuck from here on
      const int32_t n = A.op_node[k];
      int c[BL_S_MAX] = {0, 0, 0, 0, 0, 0, 0, 0};  // n's beg entries per state: they all leave now
      for (uint32_t m = live; m; m &= m - 1) {
        const int x = __ffs(m) - 1;
        if (row[x] != n) continue;
        live &= ~(1u << x);
        const int si = slot_state(A, x);
#pragma unroll
        for (int s = 0; s < BL_S_MAX; ++s) c[s] += s == si ? 1 : 0;
      }
      if (n < 0 || n >= A.NU) continue;            // counts nowhere
      const int add = A.op_kind[k] != BLANCE_OP_DEL ? A.op_state[k] : -1;
      const unsigned long long base = (unsigned long long)n * (A.S + 1), t = (unsigned long long)(r + 1);
      long long net = 0;
#pragma unroll
      for (int s = 0; s <= BL_S_MAX; ++s) {
        if (s > A.S) break;
        long long d;
        if (s < A.S) {
          d = (long long)w * ((s == add ? 1 : 0) - c[s]);
          net += d;
        } else {
          d = net;
        }
        if (d == 0) continue;
        if (MODE == 1) {
          A.ev_key[at] = ((base + s) << 32) | t;
          A.ev_val[at] = (int32_t)d;
          ++at;
        } else {
          ++n_ev;
        }
      }
    }
    if (MODE == 0) A.ev_count[p] = n_ev;
  }
}

__global__ void k_load_init(long long n, const long long* __restrict__ node_beg, long long* __restrict__ node_end,
                            unsigned long long* __restrict__ peak_key) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    node_end[i] = node_beg[i];
    peak_key[i] = pack(node_beg[i], 0);
  }
}

struct Sum {
  __host__ __device__ int32_t operator()(int32_t a, int32_t b) const { return a + b; }
};
struct SameKey {
  __host__ __device__ bool operator()(unsigned long long a, unsigned long long b) const { return (a >> 32) == (b >> 32); }
};

__global__ void k_load_peak(int n, int S, int NU, const unsigned long long* __restrict__ keys, const int32_t* __restrict__ running,
                            const long long* __restrict__ node_beg, long long* __restrict__ node_end,
                            unsigned long long* __restrict__ peak_key) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long key = keys[i], v = key >> 32;
    const long long idx = (long long)(v % (unsigned)(S + 1)) * NU + (long long)(v / (unsigned)(S + 1));
    const long long load = node_beg[idx] + running[i];
    red_max64(peak_key + idx, pack(load, (uint32_t)key));
    if (i == n - 1 || (keys[i + 1] >> 32) != v) node_end[idx] = load;   // the key's last run: its total change
  }
}

__global__ void __launch_bounds__(256) k_load_final(int S, int NU, const unsigned long long* __restrict__ peak_key,
                                                    const long long* __restrict__ node_beg, const long long* __restrict__ node_end,
                                                    long long* __restrict__ node_peak, int32_t* __restrict__ node_peak_round,
                                                    unsigned long long* __restrict__ over_key) {
  const long long n = (long long)(S + 1) * NU, row_s = (long long)S * NU;
  for (long long i0 = blockIdx.x * (long long)blockDim.x; i0 < n; i0 += (long long)gridDim.x * blockDim.x) {
    const long long i = i0 + threadIdx.x;
    unsigned long long over = 0;
    if (i < n) {
      const unsigned long long key = peak_key[i];
      const long long peak = (long long)(key >> 32) - (1ll << 31);
      node_peak[i] = peak;
      node_peak_round[i] = (int32_t)(0xFFFFFFFFu - (uint32_t)key);
      if (i >= row_s) {
        const long long q = i - row_s, o = peak - max(node_beg[i], node_end[i]);
        over = ((unsigned long long)o << 32) | (0xFFFFFFFFu - (uint32_t)q);
      }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) over = max(over, __shfl_down_sync(0xFFFFFFFFu, over, d));
    if ((threadIdx.x & 31) == 0 && over) red_max64(over_key, over);
  }
}

}  // namespace blance_load
