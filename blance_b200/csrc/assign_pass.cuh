// blance_b200/csrc/assign_pass.cuh — the hot kernel: one state pass of blance's
// greedy planner (assignStateToPartitions + findBestNodes, plan.go:98-303).
//
// The pass is a loop-carried chain: every step reads the node counts the previous
// step wrote (plan.go:286-301), so partitions are walked strictly in the
// reference's order by ONE CTA per plan instance, while the N candidate nodes of a
// step are scored in parallel.  The chain is bound by the
// latency of the serial instruction path of one step, not by memory or issue
// bandwidth, so the kernel is organised to keep that path short:
//
//   * warp specialisation: CW "compute" warps own the nodes (node n lives in compute
//     thread n % TC, register slot n / TC); one extra "service" warp streams the
//     partition records in and the new rows out, off the critical path;
//   * the partition records arrive as a LINEAR stream in step order (gathered by
//     k_gather_stream after the sort), so the service warp prefetches them with one
//     coalesced load per step, three steps ahead, into a shared-memory ring; the new
//     rows leave as a linear stream too (scattered back by k_scatter_stream);
//   * per-node state lives in REGISTERS of the owning thread (count of the state
//     being assigned as a double, all-state total, the cached "filled" term, the
//     node weight and its reciprocal); only the owner ever updates them;
//   * n2n[top][.] of the NEXT step is loaded one step early (L2, ld.cg) and patched
//     with the current step's own increments, which are fire-and-forget RED.ADDs;
//   * the score is IEEE binary64 with the reference's exact operation order
//     (plan.go:634-689), never fused with neighbouring operations.  Divisions by the
//     node weight and by P use the divisor's correctly rounded reciprocal and two
//     FMA-residual corrections (Markstein): bit-identical to the true quotient, and
//     branch-free;
//   * "sort candidates, take the first k" (plan.go:171-172, 228-229) becomes k
//     CTA-wide arg-mins of the key (ordered score bits, node position): redux.sync
//     min inside the warp, one shared-memory exchange + barrier across warps
//     (plan.go:617-628 is a strict total order, so arg-min == first of the sort);
//   * hierarchy rules (plan.go:174-226) are bit-set chains evaluated redundantly by
//     every warp (lane l owns words l, l+32, ...), so a pick costs one masked arg-min.
#pragma once

#include "pass_common.cuh"

namespace blance_dev {

struct PassSmem {
  uint4 xchg[2][32];                        // per-warp partial arg-min, double buffered
  alignas(16) int32_t ring[BL_RING][BL_REC_MAX];   // step records (pre-decoded by k_gather_stream)
  double qtab[BL_QTAB];                     // j / P for small j (plan.go:641-642)
  alignas(16) int32_t slot_bit[BL_SLP_MAX];  // 1 << (state that owns the slot), 0 for padding slots
  int32_t slot_state[BL_SLP_MAX];           // state that owns each slot
  int32_t slot_off[BL_S_MAX + 1];
  int32_t wpicks[33][BL_PICK_MAX];          // per-warp copy of the hierarchy picks
};

// CTA-wide arg-min over the compute warps.  All threads of the CTA must call; every
// thread gets the same Best.  cw = number of compute warps (they are warps 0..cw-1);
// xchg = shared address of PassSmem::xchg.
__device__ __forceinline__ Best cta_argmin(Best mine, uint32_t xchg, int& xbuf, int cw, int warp, int lane) {
  const Best w = warp_argmin(mine);
  const uint32_t base = xchg + (uint32_t)xbuf * 512u;
  if (lane == 0 && warp < cw) sts128(base + (uint32_t)warp * 16u, w.hi, w.lo, w.pos, 0u);
  __syncthreads();
  int4 e = make_int4(-1, -1, -1, 0);
  if (lane < cw) e = lds128(base + (uint32_t)lane * 16u);
  xbuf ^= 1;
  return warp_argmin(Best{(uint32_t)e.x, (uint32_t)e.y, (uint32_t)e.z});
}

#ifdef BLANCE_PASS_TIMING
#define TICK(ix) do { const long long now_ = clock64(); t_acc[ix] += now_ - t_last; t_last = now_; } while (0)
#else
#define TICK(ix) do { } while (0)
#endif

// blockDim.x = TC + 32: TC compute threads (a power of two, >= 32) + one service warp.
template <int NPT, bool HIER, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) k_assign_pass(DPool pool, int s) {
  DInst& D = pool.insts[blockIdx.x];
  if (!D.active || s >= D.S || D.pass_mode != 0) return;
  const int k = D.state_constraints[s];
  if (k <= 0) return;

  __shared__ PassSmem sm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int TC = blockDim.x - 32, cw = TC >> 5;
  const int logTC = 31 - __clz(TC);
  const bool is_service = warp == cw;
  const int N = D.N, NU = D.NU, S = D.S, SL = D.SL, SLP = D.SLP, HW = D.HW;
  const int n_assign = D.n_assign;
  const int Pn = D.P;
  const double Pd = Pn > 0 ? (double)Pn : 1.0;
  const double Py = __ddiv_rn(1.0, Pd);
  const bool has_nw = D.has_node_weights != 0;
  const int rule_lo = HIER ? D.rule_off[s] : 0, rule_hi = HIER ? D.rule_off[s + 1] : 0;

  uint32_t higher_states = 0;              // bit s2: priority[s2] < priority[s]  (plan.go:146-152)
  for (int s2 = 0; s2 < S; ++s2)
    if (D.state_priority[s2] < D.state_priority[s]) higher_states |= 1u << s2;

  const int REC = SLP + BL_REC_HDR;
  const int32_t* stream = pool.stream + D.stream_off;
  int32_t* ostream = pool.ostream + D.stream_off;
  int32_t* counts = pool.counts + D.counts_off;
  int32_t* n2n = pool.n2n + D.n2n_off;
  const int32_t* extra = (D.use_rest ? pool.extra_rest : pool.extra_first) + D.node_off;
  const uint32_t* ie_mask = pool.ie_mask + D.mask_off;

  // ---- pass constants into shared memory ------------------------------------------------
  for (int i = tid; i <= S; i += blockDim.x) sm.slot_off[i] = D.state_slot_off[i];
  for (int i = tid; i < SLP; i += blockDim.x) {
    int st = 0;
    while (st + 1 < S && i >= D.state_slot_off[st + 1]) ++st;
    sm.slot_state[i] = (i < SL) ? st : 0;
    sm.slot_bit[i] = (i < SL) ? (1 << st) : 0;
  }
  for (int i = tid; i < BL_QTAB; i += blockDim.x) sm.qtab[i] = Pn > 0 ? __ddiv_rn((double)i, Pd) : 0.0;

  // ---- per-node state in registers (compute threads) ---------------------------------------
  double cd[NPT], ff[NPT], wd[NPT], wy[NPT];   // count (as double), filled term, weight, 1/weight
  int32_t tot[NPT], qn[NPT];                   // all-state total; n2n[top][n] of the current step
  uint32_t valid_bits = 0, boost_bits = 0;
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const int n = tid + (j << logTC);
    cd[j] = 0.0; ff[j] = 0.0; wd[j] = 1.0; wy[j] = 1.0; tot[j] = 0; qn[j] = 0;
    if (!is_service && n < N) {
      int t = extra[n];
      for (int s2 = 0; s2 < S; ++s2) t += counts[s2 * N + n];
      tot[j] = t;
      cd[j] = (double)counts[s * N + n];
      if (!pool.node_removed[D.nodeid_off + n]) valid_bits |= 1u << j;
      if (has_nw && pool.node_has_weight[D.node_off + n]) {
        const int w = pool.node_weight[D.node_off + n];
        if (w > 1) { wd[j] = (double)w; wy[j] = __ddiv_rn(1.0, wd[j]); }          // plan.go:678-679 (w == 1: r / 1 == r)
        else if (w < 0 && D.booster == BLANCE_BOOSTER_CBGT_MAX) boost_bits |= 1u << j;
      }                                                                            // w == 0 / no booster: untouched (plan.go:680-682)
      if (Pn > 0) ff[j] = div_exact(__dmul_rn(0.001, (double)t), Pd, Py);          // plan.go:650
    }
  }
  // boosted nodes keep wd == wy == 1 for the (identity) division and carry -w separately
  double boost[NPT];
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const int n = tid + (j << logTC);
    boost[j] = ((boost_bits >> j) & 1u) ? -(double)pool.node_weight[D.node_off + n] : 0.0;
  }
  const bool any_boost = __syncthreads_or(boost_bits != 0) != 0;

  // ---- step-record ring, filled by the service warp from the linear stream ----------------
  int32_t rec_reg = 0, rec_reg_hi = 0;
  if (is_service) {
    for (int r = 0; r < 2 && r < n_assign; ++r) {
      if (lane < REC) sm.ring[r][lane] = stream[(size_t)r * REC + lane];
      if (lane + 32 < REC) sm.ring[r][lane + 32] = stream[(size_t)r * REC + lane + 32];
    }
    if (n_assign > 2) {
      if (lane < REC) rec_reg = stream[(size_t)2 * REC + lane];
      if (lane + 32 < REC) rec_reg_hi = stream[(size_t)2 * REC + lane + 32];
    }
  }
  __syncthreads();

  auto top_of = [&](const int32_t* rec) -> int32_t { return rec[SLP + 2]; };   // plan.go:134-138, NU stands for ""
  if (n_assign > 0 && Pn > 0) {
    const int32_t top0 = top_of(sm.ring[0]);
#pragma unroll
    for (int j = 0; j < NPT; ++j) {
      const int n = tid + (j << logTC);
      if (!is_service && n < N) qn[j] = __ldcg(n2n + (size_t)top0 * N + n);
    }
  }

  int xbuf = 0;
  constexpr int MW = (NPT + 3) / 4;
  const uint32_t sm_a = (uint32_t)__cvta_generic_to_shared(&sm);
  const uint32_t ring_a = sm_a + (uint32_t)offsetof(PassSmem, ring);
  const uint32_t xchg_a = sm_a + (uint32_t)offsetof(PassSmem, xchg);
  const uint32_t qtab_a = sm_a + (uint32_t)offsetof(PassSmem, qtab);
  const uint32_t sbit_a = sm_a + (uint32_t)offsetof(PassSmem, slot_bit);
#ifdef BLANCE_PASS_TIMING
  long long t_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  long long t_last = clock64();
#endif

  for (int i = 0; i < n_assign; ++i) {
    TICK(7);
    // ---- service warp: publish record i+2, start loading record i+3 ---------------------------
    if (is_service) {
      if (i + 2 < n_assign) {
        int32_t* dst = sm.ring[(i + 2) % BL_RING];
        if (lane < REC) dst[lane] = rec_reg;
        if (lane + 32 < REC) dst[lane + 32] = rec_reg_hi;
      }
      if (i + 3 < n_assign) {
        if (lane < REC) rec_reg = stream[(size_t)(i + 3) * REC + lane];
        if (lane + 32 < REC) rec_reg_hi = stream[(size_t)(i + 3) * REC + lane + 32];
      }
    }
    TICK(0);

    const uint32_t reca = ring_a + (uint32_t)(i % BL_RING) * (BL_REC_MAX * 4u);
    const int4 hdr = lds128(reca + (uint32_t)SLP * 4u);               // meta, w_p, top, partition
    const int32_t w_p = hdr.y;                                        // plan.go:269-275
    const int32_t top = hdr.z;
    const double stick = lds64f(reca + (uint32_t)SLP * 4u + 16u);     // plan.go:104-115

    // ---- which of my nodes does the row mention, and under which states (branch-free) ---------
    // 8 bits per node (one per state), 4 nodes per word
    uint32_t mw[MW];
#pragma unroll
    for (int w = 0; w < MW; ++w) mw[w] = 0;
    if (!is_service)
    for (int c = 0; c < (SLP >> 2); ++c) {
      const int4 v = lds128(reca + (uint32_t)c * 16u), bb = lds128(sbit_a + (uint32_t)c * 16u);
      const int32_t xs[4] = {v.x, v.y, v.z, v.w};
      const int32_t bs[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int32_t x = xs[u];
        const int jj = x >> logTC;                                    // -1 for empty slots: matches no word
        const uint32_t val = ((x & (TC - 1)) == tid) ? ((uint32_t)bs[u] << ((jj & 3) * 8)) : 0u;
#pragma unroll
        for (int w = 0; w < MW; ++w) mw[w] |= ((jj >> 2) == w) ? val : 0u;
      }
    }
    uint32_t memb[NPT];
#pragma unroll
    for (int j = 0; j < NPT; ++j) memb[j] = (mw[j >> 2] >> ((j & 3) * 8)) & 0xFFu;
    TICK(1);

    // ---- score (plan.go:634-689) and key: branch-free for the common classes --------------------
    unsigned long long key[NPT];
    uint32_t cand_bits = 0;
#pragma unroll
    for (int j = 0; j < NPT; ++j) key[j] = ~0ull;
    if (!is_service)
#pragma unroll
    for (int j = 0; j < NPT; ++j) {
      const bool cand = ((valid_bits >> j) & 1u) && !(memb[j] & higher_states);   // plan.go:142-156
      const int32_t q = qn[j];
      double qv = lds64f(qtab_a + ((uint32_t)q < BL_QTAB ? (uint32_t)q : 0u) * 8u);   // plan.go:641-642
      if ((uint32_t)q >= BL_QTAB) qv = q_over_p_slow(q, Pd, Py);
      const double base = __dadd_rn(__dadd_rn(cd[j], qv), ff[j]);                // plan.go:672-673 (+0.0 terms when P == 0)
      const double cur = ((memb[j] >> s) & 1u) ? stick : 0.0;                    // plan.go:654-662
      double r = base;
      if (has_nw) r = div_exact(r, wd[j], wy[j]);                                // plan.go:679 (identity for weight 1 / none)
      if (any_boost && ((boost_bits >> j) & 1u)) {                               // plan.go:680-681, control_test.go:19-26
        double b = boost[j];
        if (b < cur) b = cur;
        r = __dadd_rn(base, b);
      }
      r = __dsub_rn(r, cur);                                                     // plan.go:686
      // (r is never -0.0: counts convert to +0.0, x - x rounds to +0.0, and +0.0 / w = +0.0)
      key[j] = cand ? score_key(r) : ~0ull;
      cand_bits |= (cand ? 1u : 0u) << j;
    }
    TICK(2);

    int32_t qnext[NPT];
#pragma unroll
    for (int j = 0; j < NPT; ++j) qnext[j] = 0;
    int32_t top_next = NU;
    const bool have_next = (i + 1 < n_assign) && Pn > 0;
    // record i+1 is in the ring since step i-1: load n2n[top'][.] for it now (overlaps the
    // arg-min rounds) and patch it below with this step's own increments.
    if (have_next) {
      top_next = lds32(ring_a + (uint32_t)((i + 1) % BL_RING) * (BL_REC_MAX * 4u) + (uint32_t)(SLP + 2) * 4u);
#pragma unroll
      for (int j = 0; j < NPT; ++j) {
        const int n = tid + (j << logTC);
        if (!is_service && n < N) qnext[j] = __ldcg(n2n + (size_t)top_next * N + n);
      }
    }

    // arg-min over the nodes selected by `bits`; every thread calls
    auto argmin_bits = [&](uint32_t bits) -> uint32_t {
      unsigned long long bk = ~0ull;
      uint32_t bpos = 0xFFFFFFFFu;
#pragma unroll
      for (int j = 0; j < NPT; ++j)
        if (((bits >> j) & 1u) && (bpos == 0xFFFFFFFFu || key[j] < bk)) { bk = key[j]; bpos = (uint32_t)(tid + (j << logTC)); }
      return cta_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bpos}, xchg_a, xbuf, cw, warp, lane).pos;
    };
    auto mark_taken = [&](uint32_t node, uint32_t& taken_bits) {
      if ((node & (uint32_t)(TC - 1)) == (uint32_t)tid) taken_bits |= 1u << (node >> logTC);
    };

    int n_chosen = 0;
    uint32_t taken_bits = 0;
    int32_t my_choice = BLANCE_NO_NODE;      // service warp: lane c keeps the c-th chosen node

    if (HIER) {                                                                  // plan.go:174-226
      int n_picks = 0;
      uint32_t flat0 = 0xFFFFFFFEu;       // lazily computed best of the flat order ("candidateNodes[0]")
      int32_t* picks = sm.wpicks[warp];
      for (int r = rule_lo; r < rule_hi; ++r) {
        int32_t h = top;
        if (h == NU && n_picks > 0) h = picks[0];                                // plan.go:178-181
        for (int it = 0; it < k; ++it) {
          // running intersection over anchors [h] ++ picks with replace-on-empty (plan.go:743-751)
          uint32_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;
          for (int a = -1; a < n_picks; ++a) {
            const int32_t anchor = a < 0 ? h : picks[a];
            const uint32_t* res = ie_mask + ((size_t)r * (NU + 1) + anchor) * HW;
            const uint32_t r0 = lane < HW ? __ldg(res + lane) : 0u;
            const uint32_t r1 = lane + 32 < HW ? __ldg(res + lane + 32) : 0u;
            const uint32_t r2 = lane + 64 < HW ? __ldg(res + lane + 64) : 0u;
            const uint32_t r3 = lane + 96 < HW ? __ldg(res + lane + 96) : 0u;
            const bool empty = !__any_sync(0xFFFFFFFFu, (m0 | m1 | m2 | m3) != 0u);
            if (empty) { m0 = r0; m1 = r1; m2 = r2; m3 = r3; }
            else { m0 &= r0; m1 &= r1; m2 &= r2; m3 &= r3; }
          }
          uint32_t bits = 0;
#pragma unroll
          for (int j = 0; j < NPT; ++j) {
            const int wi = (tid + (j << logTC)) >> 5;         // word of my node: uniform across the warp
            const int grp = wi >> 5;
            const uint32_t word = __shfl_sync(0xFFFFFFFFu, grp == 0 ? m0 : grp == 1 ? m1 : grp == 2 ? m2 : m3, wi & 31);
            if ((word >> lane) & 1u) bits |= 1u << j;
          }
          const uint32_t best = argmin_bits(bits & cand_bits);
          uint32_t pick = best;
          if (best == 0xFFFFFFFFu) {
            if (flat0 == 0xFFFFFFFEu) flat0 = argmin_bits(cand_bits);            // plan.go:217-220
            pick = flat0;
          }
          if (pick != 0xFFFFFFFFu && n_picks < BL_PICK_MAX) {                    // plan.go:214-216
            __syncwarp();
            if (lane == 0) picks[n_picks] = (int32_t)pick;
            __syncwarp();
            ++n_picks;
          }
        }
      }
      for (int a = 0; a < n_picks && n_chosen < k; ++a) {                         // plan.go:224-229
        const uint32_t pk = (uint32_t)picks[a];
        bool dup = false;
        for (int b = 0; b < a; ++b) dup |= ((uint32_t)picks[b] == pk);
        if (dup) continue;
        if (lane == n_chosen) my_choice = (int32_t)pk;
        ++n_chosen;
        mark_taken(pk, taken_bits);
      }
    }
    while (n_chosen < k) {                                // the flat (score, position) order
      const uint32_t best = argmin_bits(cand_bits & ~taken_bits);
      if (best == 0xFFFFFFFFu) break;
      if (lane == n_chosen) my_choice = (int32_t)best;
      ++n_chosen;
      mark_taken(best, taken_bits);
    }
    TICK(3);

    // ---- apply (plan.go:238-245, 290-301) on the owners' registers -------------------------------
    const bool same_top = have_next && (top_next == top);
    uint32_t touched = taken_bits;
#pragma unroll
    for (int w = 0; w < MW; ++w) touched |= mw[w];
    if (touched)                                      // only the owners of mentioned / chosen nodes
#pragma unroll
    for (int j = 0; j < NPT; ++j) {
      const bool is_cur = (memb[j] >> s) & 1u, tk = (taken_bits >> j) & 1u;
      const int n = tid + (j << logTC);
      if ((is_cur || tk) && n < N && !is_service) {   // ids >= N (names outside nodesAll) are never scored
        int32_t t = tot[j];
        uint32_t dec = memb[j];                       // removed from every state that lists it, once per state
        const double wpd = (double)w_p;
        if ((dec >> s) & 1u) { cd[j] = __dsub_rn(cd[j], wpd); t -= w_p; dec &= ~(1u << s); }
        while (dec) {
          const int s2 = __ffs(dec) - 1;
          dec &= dec - 1;
          red_add(&counts[s2 * N + n], -w_p);        // another state's count: only the owner touches it
          t -= w_p;
        }
        if (tk) {
          cd[j] = __dadd_rn(cd[j], wpd);
          t += w_p;
          red_add(&n2n[(size_t)top * N + n], 1);    // fire-and-forget RED; re-read through L2 (ld.cg)
          if (same_top) qnext[j] += 1;                // the early load missed this increment
        }
        if (t != tot[j]) {
          tot[j] = t;
          if (Pn > 0) ff[j] = div_exact(__dmul_rn(0.001, (double)t), Pd, Py);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NPT; ++j) qn[j] = qnext[j];
    TICK(4);

    // ---- service warp: the step's outcome (chosen nodes, in order) into the output stream; the new
    // row is rebuilt from it by k_scatter_stream, in parallel, after the pass --------------------------
    if (is_service) {
      int32_t* orec = ostream + (size_t)i * REC;
      if (lane < k) orec[lane] = my_choice;            // BLANCE_NO_NODE beyond n_chosen
      if (lane == 0) orec[k] = n_chosen;               // k <= slots of the state <= SLP < REC
    }
    TICK(5);
  }
#ifdef BLANCE_PASS_TIMING
  if (lane == 0 && (warp == 0 || warp == cw) && blockIdx.x == 0)
    printf("pass s=%d warp %d steps %d cyc/step: svc-prefetch %.0f decode+memb %.0f score %.0f rounds %.0f apply %.0f svc-rowwrite %.0f loop %.0f\n",
           s, warp, n_assign, (double)t_acc[0] / n_assign, (double)t_acc[1] / n_assign, (double)t_acc[2] / n_assign,
           (double)t_acc[3] / n_assign, (double)t_acc[4] / n_assign, (double)t_acc[5] / n_assign, (double)t_acc[7] / n_assign);
#endif

  // ---- write the per-node counts of this state back ------------------------------------------------
#pragma unroll
  for (int j = 0; j < NPT; ++j) {
    const int n = tid + (j << logTC);
    if (!is_service && n < N) counts[s * N + n] = __double2int_rn(cd[j]);
  }
  if (tid == 0) D.steps += n_assign;
}

}  // namespace blance_dev
