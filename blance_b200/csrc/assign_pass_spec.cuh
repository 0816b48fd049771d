// blance_b200/csrc/assign_pass_spec.cuh — the speculative assign pass: SCOUT warps decide steps ahead of
// time from a snapshot of the node state, one LEADER warp validates and commits them in the reference's
// order and resolves the steps that move data on its own.
//
// Same chain as assign_pass.cuh / assign_pass_seq.cuh (assignStateToPartitions + findBestNodes,
// plan.go:98-303), same results.  What is different is who does the work:
//
//   * The per-node score inputs {count of the state being assigned, filled term, weight, 1/weight} live in a
//     shared-memory MIRROR that only the leader (or the whole team, on its behalf) updates.  Every update
//     belongs to an EPOCH: the leader bumps `epoch` after the update is visible and stamps the touched nodes
//     in lastchg[].
//   * The pass's step records stream into a shared-memory RING by TMA (cp.async.bulk + mbarrier), one bulk
//     copy per 32-step chunk, issued by the scout warp that owns the chunk (chunk c belongs to scout
//     c mod SW; every ring slot is only ever written by its owner).
//   * SCOUTS sweep their chunks of the ring over and over, nearest to the leader first.  For a step whose
//     partition holds exactly K clean current nodes a scout computes the K exact scores (plan.go:634-689)
//     with  nodeToNodeCounts[top][c] = qstat + A[top][c]:  qstat = the number of earlier such steps of the
//     pass with the same (top, c) pair (k_pair_rank, computed before the pass with a sort) and A = the
//     deviation from that hypothesis, a matrix that only non-sticky outcomes touch (and touching it stamps
//     the node).  It publishes {worst score T, its node, the (score, position) ranks of the K nodes, the
//     epoch it read BEFORE reading anything else} as one 16-byte word.
//   * The LEADER walks the steps 32 at a time: a published result is still exact iff none of the step's
//     current nodes was stamped after the result's epoch; the step is then STICKY - the reference's sort
//     puts exactly the current nodes first - iff T is below B0, the smallest base key (score with
//     nodeToNodeCounts = 0 and no stickiness, a lower bound of every other candidate's score; all operations
//     of plan.go:634-689 are monotone) over all live nodes.  Sticky steps change no count: the leader commits
//     the leading run of accepted steps with two fire-and-forget stores per step.
//   * The first step that is not accepted is RESOLVED by the leader alone: it keeps the smallest base keys
//     (up to 64, two per lane, unsorted) and a lower bound `ub` of every base key that is not listed.  The
//     exact scores of the listed nodes and of the partition's current nodes, K warp arg-mins, and the proof
//     that the K-th winner is below `ub` give the reference's first K nodes without looking at the other
//     nodes.  A mover updates the mirror, the matrices, the list and the epoch - about a microsecond,
//     against a CTA-wide N-way arg-min per pick in the other kernels.
//   * Every node's base key is CACHED in shared memory and rewritten by whoever changes the node.  A failed
//     proof with K winners is still the leader's: it scans the cached keys for the few nodes between ub and
//     the K-th winner and scores them too (the extended resolve).
//   * Rows that are not clean, a failed proof with too many such nodes and a list that has run dry go to the
//     TEAM: the scouts stop sweeping and run the full evaluation / the list rebuild together (named
//     barriers), exactly as the lock-step kernel would.
//
// Exactness never depends on timing: a result is only used under the two tests above, anything else falls
// through to an exact evaluation.  tools/spec_model.c checks these rules step by step inside the CPU oracle.
#pragma once

#include "assign_pass_seq.cuh"

namespace blance_dev {

#ifndef SP_LPL
#define SP_LPL 2             // list entries per leader lane
#endif
#ifndef SP_MEXT
#define SP_MEXT 7            // rebuild: entries a scout warp extracts (capped so that all fit in the list)
#endif
#define SP_D 2               // ring chunks per scout warp
#define SP_NPTS 8            // nodes per scout thread in team operations (N <= 32 * SW * SP_NPTS)
#define SP_GEN_MOD 1023      // ring generations cycle 0..1022; 1023 = never written
#ifndef SP_IDLE_NS
#define SP_IDLE_NS 500       // a scout with nothing to do sleeps this long between looks at the leader's words
#define SP_BUSY_NS 100
#endif
#ifndef SP_PINF
#define SP_PINF 1
#endif
#ifndef SP_SCAN2
#define SP_SCAN2 1
#endif
#ifndef SP_LB
// launch bound = the widest launch (12 warps); the register budget follows from it: 512 -> 128, 384 -> 168.  On
// sm_90a 128 registers spill ~180 bytes per thread; 168 keeps ~16 and is 1.9 % faster on the headline plan (H100 SXM,
// profiles/README.md).
#define SP_LB 384
#endif
#ifndef SP_U
#define SP_U 1               // groups of 32 steps the leader examines per scan (independent instruction streams)
#endif
#ifndef SP_LMIN
#define SP_LMIN 4            // rebuild the list when fewer entries are left (and it is not complete)
#endif
#ifndef SP_XMAX
#define SP_XMAX 64           // extended resolve: at most this many nodes beyond the list (SP_XMAX / 32 per leader lane); more: the team
#endif
#define SP_XPL (SP_XMAX / 32)
#ifndef SP_XRES
#define SP_XRES 1            // 0: failed proofs go to the team (no extended resolve)
#endif

enum : int { SPB_ALL = 8, SPB_GO = 9, SPB_DONE = 10, SPB_TEAM = 11 };
enum : int32_t { SP_OP_EXIT = 1, SP_OP_REBUILD = 2, SP_OP_FULL = 3 };
enum : uint32_t { SPZ_NEVER = 0x80000000u };
// leader path counts of a pass (SpecCtl::stat): team commands by cause, extended resolves
enum : int { SPS_FULL_PROOF = 0, SPS_FULL_OTHER = 1, SPS_REB_DRY = 2, SPS_FULL_MOVED = 3, SPS_XRES = 4, SPS_XOVER = 5, SPS_N = 8 };

struct SpecCtl {
  uint4 xchg[2][32];                 // team arg-min partials
  uint4 cand[32 * SP_LPL];           // rebuild: extracted {key hi, key lo, node, -}
  uint4 bound[32];                   // rebuild: per-warp lower bound of what was not extracted
  uint4 ins[16];                     // list inserts of a mover
  alignas(16) int32_t slot_bit[BL_SLP_MAX];
  alignas(8) unsigned long long mbar[32 * SP_D];
  int32_t epoch, front, cmd_seq, cmd_op, cmd_arg, cmd_epoch;
  int32_t res_n, res_same;
  int32_t res_chosen[BL_K_MAX];
  int32_t xnode[SP_XMAX];            // extended resolve: the nodes found by the scan of the base keys
  int32_t stat[SPS_N];               // leader path counts (lane 0 of the leader; SPS_*)
#ifdef BLANCE_SPEC_TIMING
  int32_t probe;                     // timing builds: a store that waits for the resolve's n2n values
#endif
};

__host__ __device__ inline size_t spec_dyn_smem_bytes(int N, int SW) {
  const size_t H = (size_t)32 * SW * SP_D;
  const size_t Np = ((size_t)N + 3) & ~(size_t)3;        // every array starts 16-byte aligned
  size_t b = Np * 32 + Np * 8 + Np * 4 + Np * 4 + ((Np + 15) & ~(size_t)15);   // mirror, base keys, totals, stamps, flags
  b += H * 64 + H * 16 + H * 16;       // records (<= 16 words), qstat, results
  return b;
}

__device__ __forceinline__ int32_t ld_relaxed_gpu(const int32_t* p) {
  int32_t v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int32_t lds32v(uint32_t a) {
  int32_t v;
  asm volatile("ld.volatile.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts32v(uint32_t a, int32_t x) {
  asm volatile("st.volatile.shared.b32 [%0], %1;" :: "r"(a), "r"(x) : "memory");
}
__device__ __forceinline__ unsigned long long lds64u(uint32_t a) {
  unsigned long long v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts64u(uint32_t a, unsigned long long x) {
  asm volatile("st.shared.b64 [%0], %1;" :: "r"(a), "l"(x) : "memory");
}
__device__ __forceinline__ void mbar_init(uint32_t a, int cnt) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(cnt) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t a, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(a), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ bool mbar_test(uint32_t a, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(a), "r"(parity) : "memory");
  return ok != 0;
}

// exact key (plan.go:634-689) with an explicit nodeToNodeCounts value q
__device__ __forceinline__ unsigned long long sp_key(double cd, double ff, double wd, double wy, bool boost, bool has_nw,
                                                     int32_t q, double cur, bool have_p, double Pd, double Py) {
  const double qv = have_p ? div_exact((double)q, Pd, Py) : 0.0;                          // plan.go:641-642
  const double base = __dadd_rn(__dadd_rn(cd, qv), ff);                                   // plan.go:672-673
  double r = base;
  if (has_nw && !boost) r = div_exact(r, wd, wy);                                         // plan.go:679
  if (boost) {                                                                            // plan.go:680-681
    double b = -wd;
    if (b < cur) b = cur;
    r = __dadd_rn(base, b);
  }
  r = __dsub_rn(r, cur);                                                                  // plan.go:686
  return score_key(r);
}

__device__ __forceinline__ bool lex_lt(unsigned long long ka, uint32_t pa, unsigned long long kb, uint32_t pb) {
  return ka < kb || (ka == kb && pa < pb);
}

// K = the state's constraints (1..BL_FAST_K).  blockDim.x = 32 * NW warps; warp 0 is the leader, the warps
// of idle_mask exit at once (they keep the leader's scheduler free), the others are the SW scouts.
template <int K>
__global__ void __launch_bounds__(SP_LB, 1) k_assign_pass_spec(DPool pool, int s, int SW, unsigned idle_mask, int /*unused*/) {
  DInst& D = pool.insts[blockIdx.x];
  if (!D.active || s >= D.S || D.pass_mode != 2) return;
  if (D.state_constraints[s] != K) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if ((idle_mask >> warp) & 1u) return;
  const bool is_leader = warp == 0;
  const int sidx = __popc(~idle_mask & ((1u << warp) - 1u)) - 1;        // scout number (leader: -1)
  const int NTA = 32 * (SW + 1), TS = 32 * SW;
  const int atid = is_leader ? lane : 32 + sidx * 32 + lane;             // rank among the active threads
  const int SWD = SW * SP_D, H = 32 * SWD;

  __shared__ SpecCtl ctl;
  extern __shared__ __align__(16) unsigned char dyn_smem[];

  const int N = D.N, S = D.S, SL = D.SL, SLP = D.SLP;
  const int n_assign = D.n_assign;
  const int lo_s = D.state_slot_off[s];
  const int Pn = D.P;
  const bool have_p = Pn > 0;
  const double Pd = have_p ? (double)Pn : 1.0;
  const double Py = __ddiv_rn(1.0, Pd);
  const bool has_nw = D.has_node_weights != 0;
  uint32_t higher_states = 0;              // bit s2: priority[s2] < priority[s]  (plan.go:146-152)
  for (int s2 = 0; s2 < S; ++s2)
    if (D.state_priority[s2] < D.state_priority[s]) higher_states |= 1u << s2;

  const int REC = SLP + BL_REC_HDR;
  const uint32_t RECB = (uint32_t)REC * 4u;
  const int32_t* stream = pool.stream + D.stream_off;
  int32_t* ostream = pool.ostream + D.stream_off;
  const int32_t* qstat_g = pool.qstat + D.part_off * 4;
  int32_t* counts = pool.counts + D.counts_off;
  int32_t* G = pool.n2n + D.n2n_off;                 // nodeToNodeCounts (plan.go:266)
  int32_t* A = pool.n2n_dev + D.n2n_off;             // its deviation from the all-sticky hypothesis
  const int32_t* extra = (D.use_rest ? pool.extra_rest : pool.extra_first) + D.node_off;

  // ---- shared memory map -------------------------------------------------------------------------------
  const uint32_t base_a = (uint32_t)__cvta_generic_to_shared(dyn_smem);
  const uint32_t Np = ((uint32_t)N + 3u) & ~3u;                  // (padded: every array starts 16-byte aligned)
  const uint32_t nd_a = base_a;                                  // mirror: {cd, ff, wd, wy} per node
  const uint32_t bk_a = nd_a + 32u * Np;                         // base keys (~0 for removed nodes and the padding)
  const uint32_t tot_a = bk_a + 8u * Np;                         // all-state totals
  const uint32_t chg_a = tot_a + 4u * Np;                        // lastchg
  const uint32_t flg_a = chg_a + 4u * Np;                        // NF_VALID | NF_BOOST
  const uint32_t rec_a = flg_a + ((Np + 15u) & ~15u);            // ring: records
  const uint32_t qs_a = rec_a + (uint32_t)H * RECB;              // ring: qstat (4 per step)
  const uint32_t dyn_a = qs_a + (uint32_t)H * 16u;               // ring: scout results
  const uint32_t ctl_a = (uint32_t)__cvta_generic_to_shared(&ctl);
  const uint32_t xchg_a = ctl_a + (uint32_t)offsetof(SpecCtl, xchg);
  const uint32_t sbit_a = ctl_a + (uint32_t)offsetof(SpecCtl, slot_bit);
  const uint32_t mbar_a = ctl_a + (uint32_t)offsetof(SpecCtl, mbar);
  const uint32_t epoch_a = ctl_a + (uint32_t)offsetof(SpecCtl, epoch);
  uint32_t front_a = ctl_a + (uint32_t)offsetof(SpecCtl, front);
#if SP_PINF
  asm volatile("" : "+r"(front_a));        // (ptxas otherwise rebuilds it from SR_CgaCtaId - an S2R - for every store of the front)
#endif
  const uint32_t seq_a = ctl_a + (uint32_t)offsetof(SpecCtl, cmd_seq);

  // ---- pass constants, mirror, ring ------------------------------------------------------------------
  for (int i = atid; i < SLP; i += NTA) {
    int st = 0;
    while (st + 1 < S && i >= D.state_slot_off[st + 1]) ++st;
    ctl.slot_bit[i] = (i < SL) ? (1 << st) : 0;
  }
  for (int n = atid; n < N; n += NTA) {
    int t = extra[n];
    for (int s2 = 0; s2 < S; ++s2) t += counts[s2 * N + n];
    const double cd = (double)counts[s * N + n];
    double wd = 1.0, wy = 1.0;
    uint32_t fl = pool.node_removed[D.nodeid_off + n] ? 0u : NF_VALID;
    if (has_nw && pool.node_has_weight[D.node_off + n]) {
      const int w = pool.node_weight[D.node_off + n];
      if (w > 1) { wd = (double)w; wy = __ddiv_rn(1.0, wd); }                          // plan.go:678-679
      else if (w < 0 && D.booster == BLANCE_BOOSTER_CBGT_MAX) { fl |= NF_BOOST; wd = (double)w; }
    }
    const double ff = have_p ? div_exact(__dmul_rn(0.001, (double)t), Pd, Py) : 0.0;   // plan.go:650
    double* nd = reinterpret_cast<double*>(dyn_smem) + 4 * (size_t)n;
    nd[0] = cd; nd[1] = ff; nd[2] = wd; nd[3] = wy;
    sts64u(bk_a + 8u * n, (fl & NF_VALID) ? sp_key(cd, ff, wd, wy, (fl & NF_BOOST) != 0, has_nw, 0, 0.0, have_p, Pd, Py) : ~0ull);
    sts32(tot_a + 4u * n, t);
    sts32(chg_a + 4u * n, 0);
    dyn_smem[(flg_a - base_a) + n] = (unsigned char)fl;
  }
  for (int n = N + atid; n < (int)Np; n += NTA) sts64u(bk_a + 8u * n, ~0ull);
  for (int i = atid; i < H; i += NTA) sts128(dyn_a + 16u * i, 0u, 0u, (uint32_t)SP_GEN_MOD << 21, 0u);
  if (atid == 0) {
    for (int i = 0; i < SWD; ++i) mbar_init(mbar_a + 8u * i, 1);
    ctl.epoch = 0; ctl.front = 0; ctl.cmd_seq = 0; ctl.cmd_op = 0; ctl.cmd_arg = 0; ctl.cmd_epoch = 0;
    ctl.res_n = 0; ctl.res_same = 0;
    for (int x = 0; x < SPS_N; ++x) ctl.stat[x] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  bar_sync(SPB_ALL, NTA);

  uint32_t slot_blocked = 0;                 // bit sl: a listed node found in slot sl of the row is not a candidate
  uint32_t slot_state_s = 0;                 //         slot sl belongs to the state being assigned
  for (int sl = 0; sl < SL && sl < 8; ++sl) {
    const uint32_t b = (uint32_t)lds32(sbit_a + 4u * sl);
    if (b & (higher_states | (1u << s))) slot_blocked |= 1u << sl;
    if (b & (1u << s)) slot_state_s |= 1u << sl;
  }

  // node owned by (scout, lane, j) in team operations: consecutive ids are spread over the warps
  auto team_node = [&](int j) { return sidx + SW * (lane + 32 * j); };
  int xbuf = 0;
  auto team_argmin = [&](Best mine) {
    const Best w = warp_argmin(mine);
    const uint32_t b = xchg_a + (uint32_t)xbuf * 512u;
    if (lane == 0) sts128(b + (uint32_t)sidx * 16u, w.hi, w.lo, w.pos, 0u);
    bar_sync(SPB_TEAM, TS);
    int4 e = make_int4(-1, -1, -1, 0);
    if (lane < SW) e = lds128(b + (uint32_t)lane * 16u);
    xbuf ^= 1;
    return warp_argmin(Best{(uint32_t)e.x, (uint32_t)e.y, (uint32_t)e.z});
  };
  const int M_ext = (32 * SP_LPL / SW) < SP_MEXT ? (32 * SP_LPL / SW) : SP_MEXT;       // rebuild: entries extracted per scout warp

  if (!is_leader) {
    // =================================== scouts ========================================================
    int chunk[SP_D];
    bool loaded[SP_D];
    int32_t seen_epoch[SP_D];                             // epoch at the last check that found slot d up to date (-1: none)
    uint32_t phase = 0;                                   // bit d: parity to wait for on slot d
    auto issue_load = [&](int d, int c) {
      if (lane == 0) {
        const int first = c * 32;
        const int nrec = (n_assign - first) < 32 ? (n_assign - first) : 32;
        const uint32_t slot0 = (uint32_t)(sidx + SW * d) * 32u;
        const uint32_t mb = mbar_a + 8u * (uint32_t)(sidx + SW * d);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(mb, (uint32_t)nrec * (RECB + 16u));
        bulk_g2s(rec_a + slot0 * RECB, stream + (size_t)first * REC, (uint32_t)nrec * RECB, mb);
        bulk_g2s(qs_a + slot0 * 16u, qstat_g + (size_t)first * 4, (uint32_t)nrec * 16u, mb);
      }
    };
#pragma unroll
    for (int d = 0; d < SP_D; ++d) {
      chunk[d] = sidx + SW * d;
      loaded[d] = false;
      seen_epoch[d] = -1;
      if (chunk[d] * 32 < n_assign) issue_load(d, chunk[d]);
    }
    int my_seq = 0;
    for (;;) {
      bool any_work = false, busy = false;
#pragma unroll
      for (int d = 0; d < SP_D; ++d) {
        // ---- a command of the leader? ----------------------------------------------------------------
        const int seq = lds32v(seq_a);
        if (seq != my_seq) {
          my_seq = seq;
          bar_sync(SPB_GO, NTA);
          const int op = *(volatile int32_t*)&ctl.cmd_op;
          if (op == SP_OP_EXIT) goto scouts_done;
          bool changed = true;
          const int32_t E1 = *(volatile int32_t*)&ctl.cmd_epoch;
          if (op == SP_OP_FULL) {
            // ---- full evaluation of step cmd_arg (the lock-step kernel's step) from the mirror --------------
            const int i = *(volatile int32_t*)&ctl.cmd_arg;
            const int ci = i >> 5;
            const uint32_t slot = (uint32_t)(ci % SWD) * 32u + (uint32_t)(i & 31);
            const uint32_t reca = rec_a + slot * RECB;
            const int4 hdr = lds128(reca + (uint32_t)SLP * 4u);               // meta, w_p, top, partition
            const int32_t w_p = hdr.y, top = hdr.z;
            const double stick = lds64f(reca + (uint32_t)SLP * 4u + 16u);
            const int n_cur = lds32(reca + (uint32_t)(SLP + 6) * 4u);
            const bool row_clean = lds32(reca + (uint32_t)(SLP + 7) * 4u) != 0;
            const bool elig = row_clean && n_cur == K;
            uint32_t memb[SP_NPTS];
            unsigned long long key[SP_NPTS];
            uint32_t cand_bits = 0, taken_bits = 0;
            int32_t frow[8];                                      // the row and the state bit of every slot, once
            uint32_t fbit[8];
            {
              const int4 r0 = lds128(reca);
              const int4 r1 = SLP > 4 ? lds128(reca + 16u) : make_int4(BLANCE_NO_NODE, BLANCE_NO_NODE, BLANCE_NO_NODE, BLANCE_NO_NODE);
              frow[0] = r0.x; frow[1] = r0.y; frow[2] = r0.z; frow[3] = r0.w;
              frow[4] = r1.x; frow[5] = r1.y; frow[6] = r1.z; frow[7] = r1.w;
#pragma unroll
              for (int sl = 0; sl < 8; ++sl) {
                fbit[sl] = sl < SLP ? (uint32_t)lds32(sbit_a + 4u * sl) : 0u;
                if (sl >= SLP) frow[sl] = -2;                     // (never a node id)
              }
            }
            int32_t qn[SP_NPTS];                                  // nodeToNodeCounts[top][n]: all loads in flight together
#pragma unroll
            for (int j = 0; j < SP_NPTS; ++j) {
              const int n = team_node(j);
              qn[j] = (have_p && n < N) ? ld_relaxed_gpu(G + (size_t)top * N + n) : 0;
            }
#pragma unroll
            for (int j = 0; j < SP_NPTS; ++j) { memb[j] = 0; key[j] = ~0ull; }
            // four node slots at a time, branch-free: four independent FP64 chains per thread in flight
#pragma unroll
            for (int h = 0; h < SP_NPTS; h += 4) {
              if (SW * 32 * h >= N) break;                                                 // (uniform)
              int4 ma[4], mb[4];
              uint32_t fl[4];
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int n = team_node(h + jj);
                const uint32_t nx = n < N ? (uint32_t)n : 0u;
                ma[jj] = lds128(nd_a + nx * 32u);
                mb[jj] = lds128(nd_a + nx * 32u + 16u);
                fl[jj] = dyn_smem[(flg_a - base_a) + nx];
              }
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = h + jj;
                const int n = team_node(j);
                uint32_t mm = 0;
#pragma unroll
                for (int sl = 0; sl < 8; ++sl)
                  if (frow[sl] == n) mm |= fbit[sl];
                const bool cand = n < N && (fl[jj] & NF_VALID) && !(mm & higher_states);   // plan.go:142-156
                const double cur = ((mm >> s) & 1u) ? stick : 0.0;                         // plan.go:654-662
                const unsigned long long k =
                    sp_key(__hiloint2double(ma[jj].y, ma[jj].x), __hiloint2double(ma[jj].w, ma[jj].z), __hiloint2double(mb[jj].y, mb[jj].x),
                           __hiloint2double(mb[jj].w, mb[jj].z), (fl[jj] & NF_BOOST) != 0, has_nw, qn[j], cur, have_p, Pd, Py);
                if (n < N) memb[j] = mm;
                if (cand) { key[j] = k; cand_bits |= 1u << j; }
              }
            }
            int n_chosen = 0;
            bool same = row_clean;
            while (n_chosen < K) {                                // the flat (score, position) order
              unsigned long long bk = ~0ull;
              uint32_t bpos = 0xFFFFFFFFu;
#pragma unroll
              for (int j = 0; j < SP_NPTS; ++j)
                if ((((cand_bits & ~taken_bits) >> j) & 1u) && (bpos == 0xFFFFFFFFu || key[j] < bk)) { bk = key[j]; bpos = (uint32_t)team_node(j); }
              const uint32_t best = team_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bpos}).pos;
              if (best == 0xFFFFFFFFu) break;
              if (sidx == 0 && lane == 0) ctl.res_chosen[n_chosen] = (int32_t)best;
              ++n_chosen;
#pragma unroll
              for (int j = 0; j < SP_NPTS; ++j)
                if ((uint32_t)team_node(j) == best) taken_bits |= 1u << j;
              bool hit = false;
              for (int q = 0; q < n_cur; ++q) hit = hit || ((uint32_t)lds32(reca + (uint32_t)(lo_s + q) * 4u) == best);
              same = same && hit;
            }
            same = same && (n_chosen == n_cur) && elig;      // (a kept short row still moves A: the hypothesis did not count it)
            if (sidx == 0 && lane == 0) { ctl.res_n = n_chosen; ctl.res_same = same ? 1 : 0; }
            changed = !same;
            // ---- apply (plan.go:238-245, 290-301) on the mirror; owners only --------------------------------
#pragma unroll
            for (int j = 0; j < SP_NPTS; ++j) {
              const int n = team_node(j);
              const bool is_cur = (memb[j] >> s) & 1u, tk = (taken_bits >> j) & 1u;
              if (n < N && (is_cur || tk)) {
                if (tk) red_add(&G[(size_t)top * N + n], 1);
                if (changed) {
                  const int dA = (tk ? 1 : 0) - ((elig && is_cur) ? 1 : 0);
                  if (dA) red_add(&A[(size_t)top * N + n], dA);
                  double* nd = reinterpret_cast<double*>(dyn_smem) + 4 * (size_t)n;
                  double cd = nd[0];
                  int32_t t0 = lds32(tot_a + 4u * n), t = t0;
                  uint32_t dec = memb[j];
                  const double wpd = (double)w_p;
                  if ((dec >> s) & 1u) { cd = __dsub_rn(cd, wpd); t -= w_p; dec &= ~(1u << s); }
                  while (dec) {
                    const int s2 = __ffs(dec) - 1;
                    dec &= dec - 1;
                    red_add(&counts[s2 * N + n], -w_p);
                    t -= w_p;
                  }
                  if (tk) { cd = __dadd_rn(cd, wpd); t += w_p; }
                  nd[0] = cd;
                  double ff = nd[1];
                  if (t != t0) {
                    sts32(tot_a + 4u * n, t);
                    if (have_p) { ff = div_exact(__dmul_rn(0.001, (double)t), Pd, Py); nd[1] = ff; }
                  }
                  const uint32_t fl = dyn_smem[(flg_a - base_a) + n];
                  sts64u(bk_a + 8u * n, (fl & NF_VALID) ? sp_key(cd, ff, nd[2], nd[3], (fl & NF_BOOST) != 0, has_nw, 0, 0.0, have_p, Pd, Py) : ~0ull);
                  sts32(chg_a + 4u * n, E1);
                }
              }
            }
            if (changed) bar_sync(SPB_TEAM, TS);          // the mirror is final before the base keys are read
          }
          if (changed) {
            // ---- rebuild: every scout warp extracts its M_ext smallest base keys and a lower bound of the rest ---
            // (from the cached base keys: whoever changes a node's mirror entry rewrites its key)
            unsigned long long bkey[SP_NPTS];
            uint32_t live = 0;
#pragma unroll
            for (int j = 0; j < SP_NPTS; ++j) {
              const int n = team_node(j);
              bkey[j] = ~0ull;
              if (n < N) {
                bkey[j] = lds64u(bk_a + 8u * (uint32_t)n);
                if (dyn_smem[(flg_a - base_a) + n] & NF_VALID) live |= 1u << j;
              }
            }
            for (int r = 0; r <= M_ext; ++r) {
              unsigned long long bk = ~0ull;
              uint32_t bpos = 0xFFFFFFFFu;
#pragma unroll
              for (int j = 0; j < SP_NPTS; ++j)
                if (((live >> j) & 1u) && (bpos == 0xFFFFFFFFu || bkey[j] < bk)) { bk = bkey[j]; bpos = (uint32_t)team_node(j); }
              const Best b = warp_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bpos});
              if (r < M_ext) {
                if (lane == 0) ctl.cand[sidx * M_ext + r] = make_uint4(b.hi, b.lo, b.pos, 0u);
#pragma unroll
                for (int j = 0; j < SP_NPTS; ++j)
                  if ((uint32_t)team_node(j) == b.pos) live &= ~(1u << j);
              } else if (lane == 0) {
                ctl.bound[sidx] = make_uint4(b.hi, b.lo, b.pos, 0u);      // all-ones when nothing is left
              }
            }
          }
          bar_sync(SPB_DONE, NTA);
        }
        // ---- my chunk of ring slot d -------------------------------------------------------------------
        int c = chunk[d];
        if (c * 32 >= n_assign) continue;
        any_work = true;
        const int fr = lds32v(front_a);
        if (fr >= (c + 1) * 32) {                       // consumed: the slot takes its next chunk
          c += SWD;
          chunk[d] = c;
          loaded[d] = false;
          seen_epoch[d] = -1;
          if (c * 32 < n_assign) issue_load(d, c);
          continue;
        }
        const uint32_t mb = mbar_a + 8u * (uint32_t)(sidx + SW * d);
        if (!loaded[d]) {
          if (!mbar_test(mb, (phase >> d) & 1u)) continue;
          loaded[d] = true;
          phase ^= 1u << d;
        }
        // ---- evaluate the chunk if one of its results is missing or out of date -----------------------------
        // (nothing is stamped without an epoch bump, so a chunk found up to date stays so until the epoch moves)
        const int32_t e0 = lds32v(epoch_a);
        if (e0 == seen_epoch[d]) continue;
        const uint32_t slot = (uint32_t)(sidx + SW * d) * 32u + (uint32_t)lane;
        const int j = c * 32 + lane;
        const uint32_t gen = (uint32_t)((c / SWD) % SP_GEN_MOD);
        const uint32_t reca = rec_a + slot * RECB;
        const bool live = j < n_assign;
        const int n_cur = lds32(reca + (uint32_t)(SLP + 6) * 4u);
        const bool clean = lds32(reca + (uint32_t)(SLP + 7) * 4u) != 0;
        const bool elig = live && clean && n_cur == K;
        int32_t cn[K];
#pragma unroll
        for (int q = 0; q < K; ++q) { cn[q] = lds32(reca + (uint32_t)(lo_s + q) * 4u); if (!elig) cn[q] = 0; }
        {
          const int4 old = lds128(dyn_a + slot * 16u);
          bool valid = (((uint32_t)old.z >> 21) & 0x3FFu) == gen;
          if (valid && elig) {
#pragma unroll
            for (int q = 0; q < K; ++q) valid = valid && lds32v(chg_a + 4u * (uint32_t)cn[q]) <= old.w;
          }
          if (!__any_sync(0xFFFFFFFFu, live && !valid)) { seen_epoch[d] = e0; continue; }
        }
        busy = true;
        const int32_t e = lds32v(epoch_a);
        __threadfence_block();                          // everything below is read after the epoch
        uint32_t z = SPZ_NEVER | (gen << 21) | 0x1FFFu;
        unsigned long long T = ~0ull;
        if (elig) {
          const int32_t top = lds32(reca + (uint32_t)(SLP + 2) * 4u);
          const double stick = lds64f(reca + (uint32_t)SLP * 4u + 16u);
          const int4 qs = lds128(qs_a + slot * 16u);
          const int32_t qsv[4] = {qs.x, qs.y, qs.z, qs.w};
          unsigned long long key[K];
          bool ok = true;
          int32_t av[K];                                        // (all loads in flight together: one L2 round trip)
#pragma unroll
          for (int q = 0; q < K; ++q) av[q] = have_p ? ld_relaxed_gpu(A + (size_t)top * N + cn[q]) : 0;
#pragma unroll
          for (int q = 0; q < K; ++q) {
            const int32_t a = av[q];
            const int4 ma = lds128(nd_a + (uint32_t)cn[q] * 32u), mb2 = lds128(nd_a + (uint32_t)cn[q] * 32u + 16u);
            const uint32_t fl = dyn_smem[(flg_a - base_a) + cn[q]];
            ok = ok && (fl & NF_VALID);
            key[q] = sp_key(__hiloint2double(ma.y, ma.x), __hiloint2double(ma.w, ma.z), __hiloint2double(mb2.y, mb2.x),
                            __hiloint2double(mb2.w, mb2.z), (fl & NF_BOOST) != 0, has_nw, qsv[q] + a, stick, have_p, Pd, Py);
          }
          if (ok) {
            int worst = 0;
            uint32_t ranks = 0;
#pragma unroll
            for (int q = 0; q < K; ++q) {
              int rank = 0;
#pragma unroll
              for (int t = 0; t < K; ++t)
                if (t != q && lex_lt(key[t], (uint32_t)cn[t], key[q], (uint32_t)cn[q])) ++rank;
              ranks = srank_pack<K>(ranks, q, rank);
              if (rank == K - 1) worst = q;
            }
            T = key[0];
            uint32_t tp = (uint32_t)cn[0];
#pragma unroll
            for (int q = 1; q < K; ++q) if (worst == q) { T = key[q]; tp = (uint32_t)cn[q]; }
            z = (gen << 21) | (ranks << 13) | tp;
          }
        }
        __threadfence_block();                          // the record (TMA) and my reads are ordered before the result
        if (live) sts128(dyn_a + slot * 16u, (uint32_t)(T >> 32), (uint32_t)T, z, (uint32_t)e);
      }
      if (!any_work) __nanosleep(SP_IDLE_NS);
      else if (!busy) __nanosleep(SP_BUSY_NS);
    }
  scouts_done:
    // ---- write the per-node counts of this state back ------------------------------------------------------
    for (int n = atid - 32; n < N; n += TS) counts[s * N + n] = __double2int_rn(reinterpret_cast<double*>(dyn_smem)[4 * (size_t)n]);
    return;
  }

  // ======================================== leader =============================================================
  unsigned long long Lk[SP_LPL];
  int32_t Ln[SP_LPL];
#pragma unroll
  for (int u = 0; u < SP_LPL; ++u) { Lk[u] = ~0ull; Ln[u] = -1; }
  unsigned long long ubk = ~0ull, B0k = ~0ull;
  uint32_t ubp = 0xFFFFFFFFu, B0p = 0xFFFFFFFFu;
  int32_t E = 0;
  int seq = 0;
  uint8_t* srank = pool.srank + D.part_off;
  long long n_fast = 0, n_res = 0, n_mov = 0, n_team = 0, n_reb = 0, n_wait = 0, n_stale = 0;
  long long cyc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, tc = clock64();   // the slots of DInst::spec_cyc
  const long long t_begin = tc;
  // path counts kept in shared memory (no leader registers): only rare paths touch them
  auto sp_bump = [&](int x) { if (lane == 0) { volatile int32_t* p = &ctl.stat[x]; *p = *p + 1; } };
#ifdef BLANCE_SPEC_TIMING
  long long cyc_n2n = 0, n_pfo = 0, cyc_x = 0;
  long long tcyc[4] = {0, 0, 0, 0};        // team cycles by cause (SPS_FULL_PROOF .. SPS_FULL_MOVED)
  int pf_next = -1;                        // the next step the last resolve's scan showed as not accepted
#define SP_PF_LOST() do { pf_next = -1; } while (0)
#else
#define SP_PF_LOST() do { } while (0)
#endif
#ifdef BLANCE_SPEC_TIMING
#define SP_T(ix) do { const long long n_ = clock64(); cyc[ix] += n_ - tc; tc = n_; } while (0)
#else
#define SP_T(ix) do { } while (0)
#endif

  auto team_cmd = [&](int op, int arg) {
    if (lane == 0) {
      *(volatile int32_t*)&ctl.cmd_op = op;
      *(volatile int32_t*)&ctl.cmd_arg = arg;
      *(volatile int32_t*)&ctl.cmd_epoch = E + 1;
      __threadfence_block();
      sts32v(seq_a, ++seq);
    } else ++seq;
    __syncwarp();
    bar_sync(SPB_GO, NTA);
    if (op != SP_OP_EXIT) bar_sync(SPB_DONE, NTA);
  };
  auto recompute_b0 = [&]() {
    unsigned long long bk = ~0ull;
    uint32_t bp = 0xFFFFFFFFu;
#pragma unroll
    for (int u = 0; u < SP_LPL; ++u)
      if (Ln[u] >= 0 && lex_lt(Lk[u], (uint32_t)Ln[u], bk, bp)) { bk = Lk[u]; bp = (uint32_t)Ln[u]; }
    const Best b = warp_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bp});
    const unsigned long long lk = ((unsigned long long)b.hi << 32) | b.lo;
    // (ub, when a mover found no room in the list, may lie below every listed key: B0 is the smaller of the two)
    if (b.pos != 0xFFFFFFFFu && lex_lt(lk, b.pos, ubk, ubp)) { B0k = lk; B0p = b.pos; }
    else { B0k = ubk; B0p = ubp; }
  };
  auto adopt_list = [&]() {                 // after a team rebuild: cand[] / bound[] -> list, ub, B0
    uint4 bb = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u);
    if (lane < SW) bb = ctl.bound[lane];
    const Best ub = warp_argmin(Best{bb.x, bb.y, bb.z});
    ubk = ((unsigned long long)ub.hi << 32) | ub.lo;
    ubp = ub.pos;
    const int n_cand = SW * M_ext;
#pragma unroll
    for (int u = 0; u < SP_LPL; ++u) {
      Lk[u] = ~0ull; Ln[u] = -1;
      const int x = lane + 32 * u;
      if (x < n_cand) {
        const uint4 c = ctl.cand[x];
        const unsigned long long k = ((unsigned long long)c.x << 32) | c.y;
        if (c.z != 0xFFFFFFFFu && lex_lt(k, c.z, ubk, ubp)) { Lk[u] = k; Ln[u] = (int32_t)c.z; }
      }
    }
    recompute_b0();
    ++n_reb;
  };
  auto publish_epoch = [&]() {
    __threadfence_block();
    __syncwarp();
    ++E;
    if (lane == 0) sts32v(epoch_a, E);
  };

  team_cmd(SP_OP_REBUILD, 0);
  adopt_list();
  SP_T(6);

  int i = 0;
  uint32_t cslot = 0, cgen = 0;
  while (i < n_assign) {
    // ---- SP_U groups of 32 steps: accept the leading run of results that are still exact and sticky --------------
    // (the ring slot and the generation of step i's chunk are carried along - cslot = (i >> 5) % SWD, cgen =
    // (i >> 5) / SWD % SP_GEN_MOD; the groups are independent instruction streams, which is what a lone warp needs)
    int4 r[SP_U];
    int32_t cn[SP_U][K];
    uint32_t reca[SP_U], okm[SP_U];
    int32_t top[SP_U];
    bool have[SP_U], never[SP_U], fresh[SP_U];
#pragma unroll
    for (int g = 0; g < SP_U; ++g) {
      const int j = i + 32 * g + lane;
      const uint32_t adv = (uint32_t)((i & 31) + lane + 32 * g) >> 5;   // chunks ahead of step i's (<= SP_U < SWD)
      uint32_t jslot = cslot + adv, gen = cgen;
      if (jslot >= (uint32_t)SWD) { jslot -= (uint32_t)SWD; if (++gen == (uint32_t)SP_GEN_MOD) gen = 0; }
      const uint32_t slot = jslot * 32u + (uint32_t)(j & 31);
      reca[g] = rec_a + slot * RECB;
      r[g] = lds128(dyn_a + slot * 16u);
#pragma unroll
      for (int q = 0; q < K; ++q) cn[g][q] = lds32(reca[g] + (uint32_t)(lo_s + q) * 4u);
      top[g] = lds32(reca[g] + (uint32_t)(SLP + 2) * 4u);               // (for the commit: not behind the ballot)
      have[g] = j < n_assign && (((uint32_t)r[g].z >> 21) & 0x3FFu) == gen;
      never[g] = ((uint32_t)r[g].z & SPZ_NEVER) != 0;
    }
#pragma unroll
    for (int g = 0; g < SP_U; ++g) {
      fresh[g] = have[g] && !never[g];
      int32_t lc[K];
#pragma unroll
      for (int q = 0; q < K; ++q) lc[q] = fresh[g] ? lds32(chg_a + 4u * (uint32_t)cn[g][q]) : 0;
#pragma unroll
      for (int q = 0; q < K; ++q) fresh[g] = fresh[g] && lc[q] <= r[g].w;
      const unsigned long long T = ((unsigned long long)(uint32_t)r[g].x << 32) | (uint32_t)r[g].y;
#if SP_SCAN2
      const bool below = lex_lt(T, (uint32_t)r[g].z & 0x1FFFu, B0k, B0p);            // (no short circuit: no branch)
      okm[g] = __ballot_sync(0xFFFFFFFFu, (int)fresh[g] & (int)below);
#else
      okm[g] = __ballot_sync(0xFFFFFFFFu, fresh[g] && lex_lt(T, (uint32_t)r[g].z & 0x1FFFu, B0k, B0p));
#endif
    }
    int32_t* Gp[SP_U][K];                                               // (address arithmetic off the ballot's shadow)
#pragma unroll
    for (int g = 0; g < SP_U; ++g) {
      const size_t row = (size_t)(uint32_t)(top[g] < 0 ? 0 : top[g]) * (size_t)N;
#pragma unroll
      for (int q = 0; q < K; ++q) Gp[g][q] = G + row + (uint32_t)(cn[g][q] < 0 ? 0 : cn[g][q]);
    }
    int run = 0;
#pragma unroll
#if SP_SCAN2
    // trailing ones of the mask = the leading run (popc on the integer pipe; ffs is a bit reverse + find-leading-one
    // on the slow pipe, and needs the all-ones case apart)
    for (int g = SP_U - 1; g >= 0; --g) run = __popc(okm[g] & ~(okm[g] + 1u)) + (okm[g] == 0xFFFFFFFFu ? run : 0);
#else
    for (int g = SP_U - 1; g >= 0; --g) run = (okm[g] == 0xFFFFFFFFu) ? 32 + run : (__ffs(~okm[g]) - 1);
#endif
#pragma unroll
    for (int g = 0; g < SP_U; ++g) {
      if (32 * g + lane < run) {                                        // commit: plan.go:238-245 and the step's outcome
#pragma unroll
        for (int q = 0; q < K; ++q)
          if (have_p) red_add(Gp[g][q], 1);
        // the outcome of an accepted step is "its current nodes in (score, position) order": one byte (0x80 | the
        // ranks, sticky_rank.cuh) in a dense array - one coalesced store per 32 steps - that k_scatter_stream expands
        srank[i + 32 * g + lane] = srank_byte((uint32_t)r[g].z >> 13);
      }
    }
    cslot += (uint32_t)((i & 31) + run) >> 5;                           // i moves on by up to SP_U chunks
    if (cslot >= (uint32_t)SWD) { cslot -= (uint32_t)SWD; if (++cgen == (uint32_t)SP_GEN_MOD) cgen = 0; }
    i += run;
    n_fast += run;
    if (run > 0 && lane == 0) sts32v(front_a, i);
    SP_T(0);
    if (run == 32 * SP_U || i >= n_assign) continue;
    // ---- step i was not accepted -----------------------------------------------------------------------------------
    bool have_l = have[0], stale_l = have[0] && !never[0] && !fresh[0];
#pragma unroll
    for (int g = 1; g < SP_U; ++g)
      if ((run >> 5) == g) { have_l = have[g]; stale_l = have[g] && !never[g] && !fresh[g]; }
    const bool have_i = __shfl_sync(0xFFFFFFFFu, (int)have_l, run & 31) != 0;
    if (!have_i) { ++n_wait; if (run == 0) __nanosleep(100); SP_T(1); continue; }        // its scout has not got there yet
    if (__shfl_sync(0xFFFFFFFFu, (int)stale_l, run & 31)) ++n_stale;
    ++n_res;
#ifdef BLANCE_SPEC_TIMING
    {
      // prefetch opportunities: the previous resolve's ballot already named this step as the next one not accepted,
      // and no team operation ran in between
      if (i == pf_next) ++n_pfo;
      uint32_t ok_i = okm[0];
#pragma unroll
      for (int g = 1; g < SP_U; ++g) if ((run >> 5) == g) ok_i = okm[g];
      const uint32_t rest = ~ok_i & ~((2u << (run & 31)) - 1u);
      pf_next = rest ? i + (__ffs(rest) - 1) - (run & 31) : -1;
    }
#endif
    {
      const uint32_t slot_i = cslot * 32u + (uint32_t)(i & 31);
      const uint32_t rb = rec_a + slot_i * RECB;
      const int4 hdr = lds128(rb + (uint32_t)SLP * 4u);               // meta, w_p, top, partition
      const int32_t w_p = hdr.y, top = hdr.z;
      const double stick = lds64f(rb + (uint32_t)SLP * 4u + 16u);
      const int n_cur = lds32(rb + (uint32_t)(SLP + 6) * 4u);
      const bool row_clean = lds32(rb + (uint32_t)(SLP + 7) * 4u) != 0;
      const int32_t myslot = lane < SLP ? lds32(rb + 4u * (uint32_t)lane) : BLANCE_NO_NODE;   // lane sl holds row[sl]
      const int32_t* Gt = G + (size_t)top * N;
      bool resolved = false;
      int n_ch = 0;
      int32_t chosen[K];
#pragma unroll
      for (int t = 0; t < K; ++t) chosen[t] = BLANCE_NO_NODE;
      bool same = false;
      if (row_clean && n_cur <= K) {
        // candidates: my listed nodes (unless the row blocks them) and, on lanes < n_cur, a current node
        unsigned long long ck[SP_LPL + 1];
        int32_t cnode[SP_LPL + 1];
        __syncwarp();                                                   // the commits above precede the loads below
#pragma unroll
        for (int u = 0; u < SP_LPL; ++u) {
          cnode[u] = Ln[u];
          ck[u] = ~0ull;
        }
        const int32_t mycur = __shfl_sync(0xFFFFFFFFu, myslot, (lo_s + (lane & 7)) & 31);
        cnode[SP_LPL] = lane < n_cur ? mycur : -1;
        ck[SP_LPL] = ~0ull;
        // row slots that block a listed node (it is current, or held by a higher-priority state)
#pragma unroll
        for (int sl = 0; sl < 8; ++sl) {
          const int32_t x = __shfl_sync(0xFFFFFFFFu, myslot, sl);
          if ((slot_blocked >> sl) & 1u) {
#pragma unroll
            for (int u = 0; u < SP_LPL; ++u) if (cnode[u] == x) cnode[u] = -1;
          }
        }
        int32_t gq[SP_LPL + 1];
#pragma unroll
        for (int u = 0; u <= SP_LPL; ++u) gq[u] = (cnode[u] >= 0 && have_p) ? ld_relaxed_gpu(Gt + cnode[u]) : 0;
#ifdef BLANCE_SPEC_TIMING
        {
          // the part of the L2 round trip that nothing overlaps (the forced wait moves the mirror loads below behind it)
          const long long t0 = clock64();
          int32_t sum = 0;
#pragma unroll
          for (int u = 0; u <= SP_LPL; ++u) sum += gq[u];
          sts32v((uint32_t)__cvta_generic_to_shared(&ctl.probe), sum);
          cyc_n2n += clock64() - t0;
        }
#endif
        bool cur_ok = true;
        {
          // branch-free over the columns: independent FP64 chains that the scheduler can interleave (a lone warp pays
          // the full latency of every dependent instruction, so the three columns one after the other cost three chains)
          int4 ma[SP_LPL + 1], mb[SP_LPL + 1];
          uint32_t fl[SP_LPL + 1];
#pragma unroll
          for (int u = 0; u <= SP_LPL; ++u) {
            const uint32_t nx = cnode[u] >= 0 ? (uint32_t)cnode[u] : 0u;
            ma[u] = lds128(nd_a + nx * 32u);
            mb[u] = lds128(nd_a + nx * 32u + 16u);
            fl[u] = dyn_smem[(flg_a - base_a) + nx];
          }
          if (cnode[SP_LPL] >= 0 && !(fl[SP_LPL] & NF_VALID)) cur_ok = false;
#pragma unroll
          for (int u = 0; u <= SP_LPL; ++u) {
            const unsigned long long k =
                sp_key(__hiloint2double(ma[u].y, ma[u].x), __hiloint2double(ma[u].w, ma[u].z), __hiloint2double(mb[u].y, mb[u].x),
                       __hiloint2double(mb[u].w, mb[u].z), (fl[u] & NF_BOOST) != 0, has_nw, gq[u], u == SP_LPL ? stick : 0.0, have_p, Pd, Py);
            ck[u] = cnode[u] >= 0 ? k : ~0ull;
          }
        }
        SP_T(2);
        if (__all_sync(0xFFFFFFFFu, cur_ok)) {
          unsigned long long lastk = 0;
          uint32_t lastp = 0;
          bool hit_all = true;
          for (int t = 0; t < K; ++t) {
            unsigned long long bk = ~0ull;
            uint32_t bp = 0xFFFFFFFFu;
#pragma unroll
            for (int u = 0; u <= SP_LPL; ++u)
              if (cnode[u] >= 0 && lex_lt(ck[u], (uint32_t)cnode[u], bk, bp)) { bk = ck[u]; bp = (uint32_t)cnode[u]; }
            const Best b = warp_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bp});
            if (b.pos == 0xFFFFFFFFu) break;
            chosen[t] = (int32_t)b.pos;
            ++n_ch;
            lastk = ((unsigned long long)b.hi << 32) | b.lo;
            lastp = b.pos;
            const bool mine_cur = cnode[SP_LPL] == (int32_t)b.pos;
            hit_all = hit_all && __any_sync(0xFFFFFFFFu, mine_cur);
#pragma unroll
            for (int u = 0; u <= SP_LPL; ++u) if (cnode[u] == (int32_t)b.pos) cnode[u] = -1;
          }
          const bool complete = ubp == 0xFFFFFFFFu;                      // every live node is listed
          if (n_ch == K) resolved = complete || lex_lt(lastk, lastp, ubk, ubp);
          else resolved = complete;
#ifdef BLANCE_SPEC_DIAG
          if (!resolved && D.debug && blockIdx.x == 0 && n_team < 24) {      // what do the failed proofs look like?
            int occ_ = 0;
#pragma unroll
            for (int u = 0; u < SP_LPL; ++u) occ_ += __popc(__ballot_sync(0xFFFFFFFFu, Ln[u] >= 0));
            const bool last_is_cur = __any_sync(0xFFFFFFFFu, lane < n_cur && mycur == (int32_t)lastp);
            if (lane == 0)
              printf("[blance] bound fail at step %d: K %d n_cur %d n_ch %d last %u (%s) key %llx ub %llx (node %u) B0 %llx listed %d hit_all %d\n",
                     i, K, n_cur, n_ch, lastp, last_is_cur ? "current" : "listed", lastk, ubk, ubp, B0k, occ_, (int)hit_all);
          }
#endif
          same = resolved && hit_all && n_ch == n_cur && n_cur == K;
          if (SP_XRES && !resolved && n_ch == K) {
            // ---- extended resolve: the proof failed, W = (lastk, lastp) is the K-th winner among listed + current --------
            // A node's exact score is never below its base key, and every node whose base key is below ub is listed.  So
            // besides the listed and the current nodes only the nodes with ub <= (base key, node) <= W can be among the
            // first K: any other node is beaten by the K candidates at or below W.  Their exact scores and K arg-mins over
            // all three groups give the step.  One pass is enough: the new K-th winner is <= W, so no node beyond the
            // set can enter.  (Listed nodes found by the scan - ub may have been lowered below them - appear twice with
            // the same key; a pick clears every entry of its node.)  More than SP_XMAX such nodes: the team evaluates
            // the step.
#ifdef BLANCE_SPEC_TIMING
            const long long tx0 = clock64();
#endif
            // the scan: lane l looks at nodes l + 32 j and sets bit j of xm for ub <= (k, n) <= W, i.e. k >= ubk (ubk + 1
            // when n < ubp) and k <= lastk (lastk - 1 when n > lastp)
            unsigned long long xm = 0;
            const unsigned long long lastk1 = lastk - 1, ubk1 = ubk + 1;
            for (int j0 = 0; 32 * j0 < N; j0 += 8) {
              unsigned long long k[8];
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {                              // (all eight loads in flight together)
                const int n = lane + 32 * (j0 + jj);
                k[jj] = lds64u(bk_a + 8u * (uint32_t)(n < N ? n : 0));
              }
              uint32_t byte = 0;
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {
                const int n = lane + 32 * (j0 + jj);
                const unsigned long long top = n <= (int)lastp ? lastk : lastk1, bot = (uint32_t)n >= ubp ? ubk : ubk1;
                byte |= (n < N && k[jj] >= bot && k[jj] <= top) ? 1u << jj : 0u;
              }
              xm |= (unsigned long long)byte << j0;
            }
            const int xc = __popcll(xm);
            int xpre = xc;                                                  // inclusive prefix sum over the lanes
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const int v = __shfl_up_sync(0xFFFFFFFFu, xpre, o);
              if (lane >= o) xpre += v;
            }
            const int cnt = __shfl_sync(0xFFFFFFFFu, xpre, 31);
            if (cnt <= SP_XMAX) {
              for (int r = xpre - xc; xm; ++r) {                            // compact: lane + 32 u takes entry u
                ctl.xnode[r] = lane + 32 * (__ffsll((long long)xm) - 1);
                xm &= xm - 1;
              }
              __syncwarp();
              int32_t xn[SP_XPL];
#pragma unroll
              for (int u = 0; u < SP_XPL; ++u) xn[u] = lane + 32 * u < cnt ? ctl.xnode[lane + 32 * u] : -1;
              // the listed and current columns as they were before the picks (a pick clears its winner's entry)
#pragma unroll
              for (int u = 0; u < SP_LPL; ++u) cnode[u] = Ln[u];
              cnode[SP_LPL] = lane < n_cur ? mycur : -1;
#pragma unroll
              for (int sl = 0; sl < 8; ++sl) {
                const int32_t x = __shfl_sync(0xFFFFFFFFu, myslot, sl);
                if ((slot_blocked >> sl) & 1u) {
#pragma unroll
                  for (int u = 0; u < SP_LPL; ++u) if (cnode[u] == x) cnode[u] = -1;
#pragma unroll
                  for (int u = 0; u < SP_XPL; ++u) if (xn[u] == x) xn[u] = -1;
                }
              }
              int32_t xq[SP_XPL];
#pragma unroll
              for (int u = 0; u < SP_XPL; ++u) xq[u] = (xn[u] >= 0 && have_p) ? ld_relaxed_gpu(Gt + xn[u]) : 0;
              unsigned long long xk[SP_XPL];
#pragma unroll
              for (int u = 0; u < SP_XPL; ++u) {
                const uint32_t nx = xn[u] >= 0 ? (uint32_t)xn[u] : 0u;
                const int4 ma = lds128(nd_a + nx * 32u), mb = lds128(nd_a + nx * 32u + 16u);
                const uint32_t fl = dyn_smem[(flg_a - base_a) + nx];
                const unsigned long long k =
                    sp_key(__hiloint2double(ma.y, ma.x), __hiloint2double(ma.w, ma.z), __hiloint2double(mb.y, mb.x),
                           __hiloint2double(mb.w, mb.z), (fl & NF_BOOST) != 0, has_nw, xq[u], 0.0, have_p, Pd, Py);
                xk[u] = xn[u] >= 0 ? k : ~0ull;
              }
              n_ch = 0;
              hit_all = true;
              for (int t = 0; t < K; ++t) {
                unsigned long long bk = ~0ull;
                uint32_t bp = 0xFFFFFFFFu;
#pragma unroll
                for (int u = 0; u <= SP_LPL; ++u)
                  if (cnode[u] >= 0 && lex_lt(ck[u], (uint32_t)cnode[u], bk, bp)) { bk = ck[u]; bp = (uint32_t)cnode[u]; }
#pragma unroll
                for (int u = 0; u < SP_XPL; ++u)
                  if (xn[u] >= 0 && lex_lt(xk[u], (uint32_t)xn[u], bk, bp)) { bk = xk[u]; bp = (uint32_t)xn[u]; }
                const Best b = warp_argmin(Best{(uint32_t)(bk >> 32), (uint32_t)bk, bp});
                chosen[t] = (int32_t)b.pos;                                 // (K candidates are at or below W)
                ++n_ch;
                hit_all = hit_all && __any_sync(0xFFFFFFFFu, cnode[SP_LPL] == (int32_t)b.pos);
#pragma unroll
                for (int u = 0; u <= SP_LPL; ++u) if (cnode[u] == (int32_t)b.pos) cnode[u] = -1;
#pragma unroll
                for (int u = 0; u < SP_XPL; ++u) if (xn[u] == (int32_t)b.pos) xn[u] = -1;
              }
              resolved = true;
              same = hit_all && n_ch == n_cur && n_cur == K;
              sp_bump(SPS_XRES);
            } else {
              sp_bump(SPS_XOVER);
            }
#ifdef BLANCE_SPEC_TIMING
            cyc_x += clock64() - tx0;
#endif
          }
        }
      }
      SP_T(3);
      if (!resolved) {
        // ---- the team evaluates the step (and rebuilds the list if a count changed) ----------------------------------
        ++n_team;
        SP_PF_LOST();
        const int why = n_ch == K ? SPS_FULL_PROOF : SPS_FULL_OTHER;     // (n_ch == K only after a failed proof)
        sp_bump(why);
#ifdef BLANCE_SPEC_TIMING
        const long long tt0 = tc;
#endif
        team_cmd(SP_OP_FULL, i);
        n_ch = *(volatile int32_t*)&ctl.res_n;
        same = *(volatile int32_t*)&ctl.res_same != 0;
#pragma unroll
        for (int t = 0; t < K; ++t) chosen[t] = t < n_ch ? *(volatile int32_t*)&ctl.res_chosen[t] : BLANCE_NO_NODE;
        int32_t* orec = ostream + (size_t)i * REC;
        if (lane == 0) {
#pragma unroll
          for (int t = 0; t < K; ++t) orec[t] = chosen[t];
          orec[K] = n_ch;
        }
        if (!same) { adopt_list(); publish_epoch(); ++n_mov; sp_bump(SPS_FULL_MOVED); }
        SP_T(6);
#ifdef BLANCE_SPEC_TIMING
        tcyc[why] += tc - tt0;
        if (!same) tcyc[SPS_FULL_MOVED] += tc - tt0;
#endif
      } else {
        int32_t* orec = ostream + (size_t)i * REC;
        if (lane == 0) {
#pragma unroll
          for (int t = 0; t < K; ++t) orec[t] = chosen[t];
          orec[K] = n_ch;
        }
        if (lane < n_ch && have_p) {
          int32_t mine = chosen[0];
#pragma unroll
          for (int t = 1; t < K; ++t) if (lane == t) mine = chosen[t];
          red_add(&G[(size_t)top * N + mine], 1);                      // plan.go:238-245
        }
        if (!same) {
          // ---- a mover: lanes 0..n_cur-1 take the old nodes, lanes 8..8+n_ch-1 the new ones -------------------------
          ++n_mov;
          const int32_t E1 = E + 1;
          const bool elig = n_cur == K;
          // A[top][x] changes by (x is chosen) - (the hypothesis counted x: eligible row and x current); a node whose
          // count or A entry changes is stamped, so results computed from the old values are rejected
          int delta = 0, dA = 0;
          const int32_t oldx = __shfl_sync(0xFFFFFFFFu, myslot, (lo_s + (lane & 7)) & 31);
          int32_t newx = chosen[0];
#pragma unroll
          for (int t = 1; t < K; ++t) if (lane - 8 == t) newx = chosen[t];
          const bool is_old = lane < n_cur, is_new = lane >= 8 && lane < 8 + n_ch;
          const int32_t x = is_old ? oldx : (is_new ? newx : -1);
          bool again = false;                   // old node that is chosen again / new node that was current
          if (is_old) {
#pragma unroll
            for (int t = 0; t < K; ++t) again = again || (t < n_ch && chosen[t] == x);
          }
          uint32_t memb = 0;                    // states (other than s) whose list holds my new node
#pragma unroll
          for (int sl = 0; sl < 8; ++sl) {
            const int32_t y = __shfl_sync(0xFFFFFFFFu, myslot, sl);
            if (is_new && y == x && sl < SLP) {
              if ((slot_state_s >> sl) & 1u) again = true;
              else memb |= (uint32_t)lds32(sbit_a + 4u * sl);
            }
          }
          bool act = false;
          if (is_old && !again) { act = true; delta = -w_p; dA = elig ? -1 : 0; }
          if (is_new && !again) { act = true; delta = w_p; dA = 1; }
          if (is_new && again && !elig) { act = true; dA = 1; memb = 0; }      // kept node of a short row: only A moves
          act = act && x >= 0;
          unsigned long long nk = ~0ull;
          bool ins = false;
          if (act) {
            if (have_p && dA) red_add(&A[(size_t)top * N + x], dA);
            const int4 ma = lds128(nd_a + (uint32_t)x * 32u), mb = lds128(nd_a + (uint32_t)x * 32u + 16u);
            const uint32_t fl = dyn_smem[(flg_a - base_a) + x];
            double cd = __hiloint2double(ma.y, ma.x), ff = __hiloint2double(ma.w, ma.z);
            cd = __dadd_rn(cd, (double)delta);
            int32_t t0 = lds32(tot_a + 4u * (uint32_t)x), t = t0 + delta;
            while (memb) {
              const int s2 = __ffs(memb) - 1;
              memb &= memb - 1;
              red_add(&counts[s2 * N + x], -w_p);
              t -= w_p;
            }
            if (t != t0) {
              sts32(tot_a + 4u * (uint32_t)x, t);
              if (have_p) ff = div_exact(__dmul_rn(0.001, (double)t), Pd, Py);
            }
            double* nd = reinterpret_cast<double*>(dyn_smem) + 4 * (size_t)x;
            nd[0] = cd; nd[1] = ff;
            sts32(chg_a + 4u * (uint32_t)x, E1);
            nk = sp_key(cd, ff, __hiloint2double(mb.y, mb.x), __hiloint2double(mb.w, mb.z), (fl & NF_BOOST) != 0, has_nw, 0, 0.0, have_p, Pd, Py);
            sts64u(bk_a + 8u * (uint32_t)x, (fl & NF_VALID) ? nk : ~0ull);
            ins = (fl & NF_VALID) && lex_lt(nk, (uint32_t)x, ubk, ubp);
          }
          __syncwarp();
          SP_T(4);
          // list: drop the touched nodes, take the ones that are (still) below ub into free places
#pragma unroll
          for (int u = 0; u < SP_LPL; ++u)
            if (Ln[u] >= 0 && lds32(chg_a + 4u * (uint32_t)Ln[u]) == E1) { Ln[u] = -1; Lk[u] = ~0ull; }
          const uint32_t insm = __ballot_sync(0xFFFFFFFFu, ins);
          const int n_ins = __popc(insm);
          if (n_ins) {
            if (ins) ctl.ins[__popc(insm & ((1u << lane) - 1u))] = make_uint4((uint32_t)(nk >> 32), (uint32_t)nk, (uint32_t)x, 0u);
            __syncwarp();
            int placed = 0;
#pragma unroll
            for (int u = 0; u < SP_LPL; ++u) {
              const uint32_t freem = __ballot_sync(0xFFFFFFFFu, Ln[u] < 0);
              const int r2 = placed + __popc(freem & ((1u << lane) - 1u));
              if (Ln[u] < 0 && r2 < n_ins) {
                const uint4 e = ctl.ins[r2];
                Lk[u] = ((unsigned long long)e.x << 32) | e.y;
                Ln[u] = (int32_t)e.z;
              }
              placed += __popc(freem);
            }
            for (int r2 = placed; r2 < n_ins; ++r2) {                  // no room: the node stays unlisted, ub covers it
              const uint4 e = ctl.ins[r2];
              const unsigned long long k = ((unsigned long long)e.x << 32) | e.y;
              if (lex_lt(k, e.z, ubk, ubp)) { ubk = k; ubp = e.z; }
            }
            __syncwarp();
          }
          int occ = 0;
#pragma unroll
          for (int u = 0; u < SP_LPL; ++u) occ += __popc(__ballot_sync(0xFFFFFFFFu, Ln[u] >= 0));
          if (occ < SP_LMIN && ubp != 0xFFFFFFFFu) {
            publish_epoch();
            SP_T(5);
            SP_PF_LOST();
            sp_bump(SPS_REB_DRY);
#ifdef BLANCE_SPEC_TIMING
            const long long tt0 = tc;
#endif
            team_cmd(SP_OP_REBUILD, 0);                                 // reads the base keys only
            adopt_list();
            SP_T(6);
#ifdef BLANCE_SPEC_TIMING
            tcyc[SPS_REB_DRY] += tc - tt0;
#endif
          } else {
            recompute_b0();
            publish_epoch();
            SP_T(5);
          }
        }
      }
      if ((++i & 31) == 0) {
        if (++cslot == (uint32_t)SWD) { cslot = 0; if (++cgen == (uint32_t)SP_GEN_MOD) cgen = 0; }
      }
      if (lane == 0) sts32v(front_a, i);
    }
  }
  team_cmd(SP_OP_EXIT, 0);
  if (lane == 0) {
    D.steps += n_assign;
    D.fast_steps += n_fast;
    D.spec_resolved += n_res; D.spec_movers += n_mov; D.spec_team += n_team; D.spec_rebuilds += n_reb;
    D.spec_waits += n_wait; D.spec_stale += n_stale;
#ifdef BLANCE_SPEC_DIAG
    if (D.debug && blockIdx.x == 0)
      printf("[blance] spec pass state %d K %d: steps %d accepted %lld resolved %lld movers %lld team %lld rebuilds %lld stale %lld waits %lld\n",
             s, K, n_assign, n_fast, n_res, n_mov, n_team, n_reb, n_stale, n_wait);
#endif
    cyc[7] = clock64() - t_begin;
    for (int x = 0; x < 8; ++x) D.spec_cyc[x] += cyc[x];
    for (int x = 0; x < 6; ++x) D.spec_path[x] += *(volatile int32_t*)&ctl.stat[x];
#ifdef BLANCE_SPEC_TIMING
    D.spec_cyc_n2n += cyc_n2n;
    D.spec_pf_opp += n_pfo;
    D.spec_cyc_x += cyc_x;
    for (int x = 0; x < 4; ++x) D.spec_cyc_team[x] += tcyc[x];
#endif
  }
#undef SP_T
#undef SP_PF_LOST
}

}  // namespace blance_dev
