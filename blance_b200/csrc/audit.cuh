// blance_b200/csrc/audit.cuh — the audit of a partition map (include/blance_b200.h, "auditing a partition map"):
// unmet constraints, fault-domain exposure and failover spread (k_map_audit, one thread per partition), hierarchy-rule
// misses (k_map_audit_rules, one warp per partition, lanes over the words of the bit sets; launched only when an
// instance has rules) and the largest entry of the failover matrix (k_audit_n2n_max).  Grid: x strides over the
// partitions of instance blockIdx.y, as k_scenario_summary.
#pragma once

#include <cuda_runtime.h>

#include "blance_b200.h"
#include "device_types.cuh"

namespace blance_dev {

#define AUDIT_DEPTH_MAX 16     // edges from a vertex to its root
#define AUDIT_RULES_MAX 256    // rules of one instance (8 states x 32)
#define AUDIT_HW_LANE 4        // mask words per lane: hier_words <= 128

// One audited map.  A partition reads `rows` / `meta`; when `pflags` is given (the final map of a plan) a partition
// without PF_IN_ASSIGN reads `alt_rows` / `alt_meta` if it has PF_IN_PREV and has no lists otherwise.  Shapes are the
// 2-bit fields of `meta`, or, when meta is NULL, the caller's bytes shape8[p][S].
struct AuditInst {
  const int32_t* rows; const int32_t* alt_rows;
  const uint32_t* meta; const uint32_t* alt_meta;
  const uint8_t* shape8;
  const uint8_t* pflags;
  const uint32_t* ie_mask;        // [n_rules][NU + 1][HW]
  const int32_t* dom_parent;      // [V] or NULL (nodes only)
  long long* out;                 // short[S] | over[S] | miss[Rc] | tested[Rc] | dom_top[V] | dom_all[V] | dom_copies[V] |
                                  // short_parts, rule_miss_parts, no_top_parts, n2n key
  int32_t* n2n;                   // [N][N] or NULL
  uint8_t* part_flags;            // [P] or NULL
  int32_t stride;                 // int32 per row
  int32_t P, N, NU, V, S, top_state, HW, n_rules, Rc;
  int32_t constraints[BL_S_MAX], slot_off[BL_S_MAX + 1], rule_off[BL_S_MAX + 1];
};

__host__ __device__ inline long long audit_out_words(int S, int Rc, int V) { return 2ll * S + 2ll * Rc + 3ll * V + 4; }

// atomics whose result nobody reads: red.* (an atomicAdd with an unused result may compile to ATOMG ... RZ and hold a
// scoreboard for the L2 round trip)
__device__ __forceinline__ void red_add64(long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add32(int32_t* p, int32_t v) {
  asm volatile("red.relaxed.gpu.global.add.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_max64(long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void reds_add32(uint32_t* p, uint32_t v) {
  asm volatile("red.shared.add.u32 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}

// the row and the shape word (2 bits per state) partition p reads
__device__ __forceinline__ const int32_t* audit_row(const AuditInst& A, long long p, uint32_t* shapes) {
  const int32_t* row = A.rows + p * A.stride;
  uint32_t m = 0;
  if (A.meta) m = A.meta[p] & 0xFFFFu;
  else for (int s = 0; s < A.S; ++s) m |= (uint32_t)(A.shape8[p * A.S + s] & 3u) << (2 * s);
  if (A.pflags) {
    const uint8_t f = A.pflags[p];
    if (!(f & PF_IN_ASSIGN)) {
      row = A.alt_rows + p * A.stride;
      m = (f & PF_IN_PREV) ? (A.alt_meta[p] & 0xFFFFu) : 0u;
    }
  }
  *shapes = m;
  return row;
}

__device__ __forceinline__ int audit_parent(const AuditInst& A, int v) { return A.dom_parent ? __ldg(A.dom_parent + v) : -1; }

__device__ __forceinline__ int audit_depth(const AuditInst& A, int v) {
  int d = 0;
  for (int u = audit_parent(A, v); u >= 0 && d < AUDIT_DEPTH_MAX; u = audit_parent(A, u)) ++d;
  return d;
}

// deepest common ancestor of two vertices, -1 when they are in different trees
__device__ __forceinline__ int audit_dca(const AuditInst& A, int a, int b) {
  if (a == b || !A.dom_parent) return a == b ? a : -1;
  int da = audit_depth(A, a), db = audit_depth(A, b);
  for (; da > db; --da) a = audit_parent(A, a);
  for (; db > da; --db) b = audit_parent(A, b);
  for (int i = 0; a != b && i <= AUDIT_DEPTH_MAX; ++i) {
    a = audit_parent(A, a); b = audit_parent(A, b);
    if (a < 0 || b < 0) return -1;
  }
  return a == b ? a : -1;
}

// Constraints, fault domains, failover spread.  SMEM: the per-vertex tables of one instance live in shared memory
// (u32 [3][V]) and are flushed once per CTA; the per-state tables (u32 [2][S]) always do.
template <bool SMEM>
__global__ void k_map_audit(const AuditInst* __restrict__ insts) {
  extern __shared__ uint32_t s_dom[];
  __shared__ uint32_t s_state[2 * BL_S_MAX];
  const AuditInst& A = insts[blockIdx.y];
  const int S = A.S, V = A.V, NU = A.NU, N = A.N;
  long long* o_state = A.out;
  long long* o_dom = A.out + 2ll * S + 2ll * A.Rc;
  long long* o_scal = o_dom + 3ll * V;
  if (threadIdx.x < 2 * BL_S_MAX) s_state[threadIdx.x] = 0;
  if (SMEM) for (int x = threadIdx.x; x < 3 * V; x += blockDim.x) s_dom[x] = 0;
  __syncthreads();
  auto dom_add = [&](int table, int v) {
    if (SMEM) reds_add32(&s_dom[table * V + v], 1u);
    else red_add64(&o_dom[(long long)table * V + v], 1ull);
  };
  uint32_t n_short = 0, n_notop = 0;
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < A.P; p += (long long)gridDim.x * blockDim.x) {
    uint32_t shapes;
    const int32_t* row = audit_row(A, p, &shapes);
    int h = -1;
    if (meta_shape(shapes, A.top_state) == BLANCE_SHAPE_LIST && A.slot_off[A.top_state + 1] > A.slot_off[A.top_state])
      h = row[A.slot_off[A.top_state]];
    if (h >= NU) h = -1;
    bool is_short = false;
    int dca = -2;                                   // -2: no copy yet, -1: copies in different trees
    for (int s = 0; s < S; ++s) {
      if (meta_shape(shapes, s) == BLANCE_SHAPE_ABSENT) continue;
      int len = 0;
      const int end = meta_shape(shapes, s) == BLANCE_SHAPE_LIST ? A.slot_off[s + 1] : A.slot_off[s];     // a nil slice has no nodes
      for (int c = A.slot_off[s]; c < end; ++c, ++len) {
        const int32_t x = row[c];
        if (x == BLANCE_NO_NODE) break;
        if (x < 0 || x >= NU) continue;
        for (int v = x, d = 0; v >= 0 && d <= AUDIT_DEPTH_MAX; v = audit_parent(A, v), ++d) dom_add(2, v);
        dca = dca == -2 ? x : dca == -1 ? -1 : audit_dca(A, dca, x);
        if (A.n2n && h >= 0 && h < N && x < N && x != h) red_add32(A.n2n + (long long)h * N + x, 1);
      }
      const int k = A.constraints[s];
      if (k <= 0) continue;
      if (len < k) { reds_add32(&s_state[s], (uint32_t)(k - len)); is_short = true; }
      if (len > k) reds_add32(&s_state[BL_S_MAX + s], (uint32_t)(len - k));
    }
    for (int v = h, d = 0; v >= 0 && d <= AUDIT_DEPTH_MAX; v = audit_parent(A, v), ++d) dom_add(0, v);
    for (int v = dca, d = 0; v >= 0 && d <= AUDIT_DEPTH_MAX; v = audit_parent(A, v), ++d) dom_add(1, v);
    n_short += is_short ? 1u : 0u;
    n_notop += h < 0 ? 1u : 0u;
    if (A.part_flags) A.part_flags[p] = (uint8_t)((is_short ? 1 : 0) | (h < 0 ? 4 : 0));
  }
  // warp-aggregated scalars: one RED per warp and counter
  n_short = __reduce_add_sync(0xFFFFFFFFu, n_short);
  n_notop = __reduce_add_sync(0xFFFFFFFFu, n_notop);
  if ((threadIdx.x & 31) == 0) {
    if (n_short) red_add64(&o_scal[0], n_short);
    if (n_notop) red_add64(&o_scal[2], n_notop);
  }
  __syncthreads();
  if (threadIdx.x < 2 * BL_S_MAX && s_state[threadIdx.x]) {
    const int t = threadIdx.x / BL_S_MAX, s = threadIdx.x % BL_S_MAX;
    if (s < S) red_add64(&o_state[(long long)t * S + s], s_state[threadIdx.x]);
  }
  if (SMEM)
    for (int x = threadIdx.x; x < 3 * V; x += blockDim.x)
      if (s_dom[x]) red_add64(&o_dom[x], s_dom[x]);
}

// Hierarchy rules: one warp per partition.  Lane l holds words l, l + 32, l + 64, l + 96 of the running intersection;
// its emptiness (plan.go:746) is one redux.sync.or.  Indices are clamped and results selected, so that the warp stays
// converged through the shuffles.  Runs after k_map_audit on the same stream (it ORs bit 1 into part_flags).
__global__ void k_map_audit_rules(const AuditInst* __restrict__ insts) {
  __shared__ uint32_t s_rule[2 * AUDIT_RULES_MAX];
  const AuditInst& A = insts[blockIdx.y];
  if (A.n_rules <= 0) return;
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int S = A.S, NU = A.NU, HW = A.HW;
  long long* o_rule = A.out + 2ll * S;
  long long* o_scal = A.out + 2ll * S + 2ll * A.Rc + 3ll * A.V;
  for (int x = threadIdx.x; x < 2 * AUDIT_RULES_MAX; x += blockDim.x) s_rule[x] = 0;
  __syncthreads();
  uint32_t n_miss_parts = 0;                        // lane 0 counts
  for (long long p = blockIdx.x * (long long)wpb + (threadIdx.x >> 5); p < A.P; p += (long long)gridDim.x * wpb) {
    uint32_t shapes;
    const int32_t* row = audit_row(A, p, &shapes);
    const int32_t mine = lane < A.stride ? row[lane] : BLANCE_NO_NODE;     // a row is at most 32 slots
    int h = NU;
    if (meta_shape(shapes, A.top_state) == BLANCE_SHAPE_LIST && A.slot_off[A.top_state + 1] > A.slot_off[A.top_state]) {
      const int32_t t = __shfl_sync(full, mine, A.slot_off[A.top_state]);
      h = (t >= 0 && t < NU) ? t : NU;
    }
    bool missed = false;
    for (int s = 0; s < S; ++s) {
      const int lo = A.slot_off[s], hi = A.slot_off[s + 1], k = A.constraints[s];
      if (A.rule_off[s + 1] <= A.rule_off[s] || k <= 0 || meta_shape(shapes, s) != BLANCE_SHAPE_LIST) continue;     // absent or nil: nothing to test
      const unsigned gaps = __ballot_sync(full, lane >= lo && lane < hi && mine == BLANCE_NO_NODE) | (hi < 32 ? full << hi : 0u);
      const int len = (gaps ? __ffs(gaps) - 1 : 32) - lo;
      const int n_test = min(len, k);
      for (int r = A.rule_off[s]; r < A.rule_off[s + 1]; ++r) {
        const uint32_t* mask = A.ie_mask + (long long)r * (NU + 1) * HW;
        uint32_t rv[AUDIT_HW_LANE];
#pragma unroll
        for (int i = 0; i < AUDIT_HW_LANE; ++i) rv[i] = 0;
        uint32_t tested = 0, miss = 0;
        for (int j = 0; j < n_test; ++j) {
          // the node this position adds to the prefix: the anchor at j = 0, L_s[j-1] after it; with h = "" the
          // prefix of j > 0 starts over from L_s[0] (plan.go:178-181)
          int y = j == 0 ? h : __shfl_sync(full, mine, lo + j - 1);
          y = (y >= 0 && y < NU) ? y : NU;       // an id outside [0, n_node_ids) (the header forbids it) reads the "" row
          const bool restart = j == 1 && h == NU;
          uint32_t any = 0;
#pragma unroll
          for (int i = 0; i < AUDIT_HW_LANE; ++i) { rv[i] = restart ? 0u : rv[i]; any |= rv[i]; }
          const bool empty = __reduce_or_sync(full, any) == 0;
#pragma unroll
          for (int i = 0; i < AUDIT_HW_LANE; ++i) {
            const int w = lane + 32 * i;
            const uint32_t res = w < HW ? __ldg(mask + (long long)y * HW + w) : 0u;
            rv[i] = empty ? res : (rv[i] & res);
          }
          if (j == 0 && s == A.top_state) continue;                 // the anchor itself
          const int x = __shfl_sync(full, mine, lo + j);
          uint32_t hit = 0;
#pragma unroll
          for (int i = 0; i < AUDIT_HW_LANE; ++i) hit |= (lane + 32 * i == (x >> 5)) ? (rv[i] >> (x & 31)) & 1u : 0u;
          const bool ok = x >= 0 && x < A.N && __reduce_or_sync(full, hit) != 0;
          ++tested;
          miss += ok ? 0u : 1u;
        }
        if (lane == 0) {
          if (tested) reds_add32(&s_rule[AUDIT_RULES_MAX + r], tested);
          if (miss) reds_add32(&s_rule[r], miss);
        }
        missed |= miss != 0;
      }
    }
    if (lane == 0 && missed) {
      ++n_miss_parts;
      if (A.part_flags) A.part_flags[p] |= 2;
    }
  }
  if (lane == 0 && n_miss_parts) red_add64(&o_scal[1], n_miss_parts);
  __syncthreads();
  for (int x = threadIdx.x; x < 2 * AUDIT_RULES_MAX; x += blockDim.x) {
    const int t = x / AUDIT_RULES_MAX, r = x % AUDIT_RULES_MAX;
    if (s_rule[x] && r < A.n_rules) red_add64(&o_rule[(long long)t * A.Rc + r], s_rule[x]);
  }
}

// The largest entry of each instance's failover matrix and the lowest (a, b) that holds it, as one u64 key
// count << 32 | ~index (the matrix has at most 2^26 entries), reduced per warp and then with one RED.MAX.
__global__ void k_audit_n2n_max(const AuditInst* __restrict__ insts) {
  const AuditInst& A = insts[blockIdx.y];
  if (!A.n2n) return;
  const long long n = (long long)A.N * A.N;
  unsigned long long best = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t c = (uint32_t)A.n2n[i];
    const unsigned long long key = ((unsigned long long)c << 32) | (0xFFFFFFFFu - (uint32_t)i);
    best = (c && key > best) ? key : best;
  }
  const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(best >> 32));
  const uint32_t lo = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(best >> 32) == hi ? (uint32_t)best : 0u);
  if ((threadIdx.x & 31) == 0 && hi)
    red_max64(A.out + 2ll * A.S + 2ll * A.Rc + 3ll * A.V + 3, ((unsigned long long)hi << 32) | lo);
}

}  // namespace blance_dev
