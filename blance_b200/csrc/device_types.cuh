// blance_b200/csrc/device_types.cuh — device-side data layout of a batch of plans.
//
// All instances of a batch live in ONE set of pooled arrays; instance i owns the
// slices named by the offsets in its DInst.  A single PlanNextMapEx call is a
// batch of one.  Layout in HBM (sizes for the 1M x 1024 workload in DESIGN.md):
//
//   rows / prev_rows   int32 [sum PU_i][SLP_i]   rows padded to SLP = round_up(SL,4) so a
//                                                row is one or two 16-byte vectors
//   pmeta / prev_meta  uint32[sum PU_i]          2 shape bits per state (bits 0..15),
//                                                warn bit per state (bits 16..23)
//   pflags             uint8 [sum PU_i]          IN_PREV | IN_ASSIGN | HAS_WEIGHT
//   pweight, name_rank int32 [sum PU_i]
//   keys / order       uint64 / int32 [sum PU_i] partition sort key and permutation
//   stream / ostream   int32 [sum PU_i][SLP_i+8] the pass's input / output records in STEP order
//                                                (row | meta, w_p, top, partition | stickiness)
//   counts             int32 [S_i][N_i]          stateNodeCounts (plan.go:92-94)
//   n2n                int32 [NU_i+1][N_i]       nodeToNodeCounts (plan.go:266), row NU = ""
//   n2n_dev            int32 [NU_i+1][N_i]       speculative pass: n2n minus the all-sticky hypothesis
//   qstat              int32 [sum PU_i][4]       speculative pass: per step and current node, the number of
//                                                earlier eligible steps with the same (top, node) pair
//   pair_keys / vals   uint64 / uint32 [4 sum PU_i] (x2) the pair sort behind qstat
//   ie_mask            uint32[R_i][NU_i+1][HW_i] hierarchy include/exclude bit sets
#pragma once

#include <cstdint>

#define BL_S_MAX 8        // states per model
#define BL_K_MAX 16       // constraints per state
#define BL_SLP_MAX 32     // padded slots per row
#define BL_PICK_MAX 32    // hierarchy picks per step (rules x constraints)
#define BL_RING 8         // step-record ring depth in shared memory (records i .. i+3 live, i+4 in flight)

// node_removed on the device: bit 0 = in nodesToRemove, bit 1 = outside this plan's nodesAll (a chain stage's
// membership mask, blance_plan_chains).  Candidate tests read "!= 0"; the strip of plan.go:83-88 and the bucket-0
// test of plan.go:544 read bit 0 only.  A caller's table is normalised to 0 / 1 when it is staged.
enum : uint8_t { NR_REMOVE = 1, NR_OUTSIDE = 2 };

enum : uint8_t { PF_IN_PREV = 1, PF_IN_ASSIGN = 2, PF_HAS_WEIGHT = 4,
                 PF_PREV_EXTRA = 8 };   // the prevMap entry has keys outside the model (until plan.go:49-52 replaces it)

struct DInst {
  // static scalars
  int32_t N, NU, S, PU, SL, SLP, HW, n_rules;
  int32_t top_state, booster, has_part_weights, has_node_weights, has_hier_rules;
  int32_t max_iters, n_assign, n_valid, engine;
  int32_t debug;           // BLANCE_SPEC_STATS: the speculative kernel prints its counters after every pass
  int32_t state_priority[BL_S_MAX], state_constraints[BL_S_MAX], state_slot_off[BL_S_MAX + 1];
  int32_t state_stickiness[BL_S_MAX], state_has_stickiness[BL_S_MAX], rule_off[BL_S_MAX + 1];
  // offsets (in elements) into the pooled arrays
  int64_t part_off, rows_off, node_off, nodeid_off, counts_off, n2n_off, mask_off, stream_off;
  // dynamic state of the convergence loop (plan.go:32-56)
  int32_t P;               // len(prevMap) seen by this iteration (plan.go:161)
  int32_t rm_active;       // len(nodesToRemove) > 0 (iteration 1 only, plan.go:54)
  int32_t add_active;      // nodesToAdd may be non-empty (iteration 1 only, plan.go:55)
  int32_t add_is_nil;      // nodesToAdd == nil (plan.go:554)
  int32_t use_rest;        // extra_tot_rest instead of extra_tot_first
  int32_t active, converged, iters_run, mismatch;
  int32_t pass_mode;       // kernel of the current pass: 0 lock-step (assign_pass.cuh), 1 sequencer (assign_pass_seq.cuh),
                           // 2 speculative (assign_pass_spec.cuh)
  int32_t n_elig;          // rows of the current pass that hold exactly k clean current nodes (k_gather_stream)
  int32_t n_clean;         // rows of the current pass that are clean and hold at most k current nodes
  long long steps;
  long long fast_steps;    // steps decided without a full evaluation (sequencer windows / accepted scout results)
  // counters of the speculative kernel (whole plan)
  long long spec_resolved, spec_movers, spec_team, spec_rebuilds, spec_waits, spec_stale;
  long long spec_cyc[8];   // leader cycles: scans | waits | resolve loads+keys | resolve picks | mover mirror | mover list+publish | team | passes
  long long spec_cyc_n2n;  // of resolve loads+keys: the cycles spent waiting for the n2n values (timing builds)
  long long spec_pf_opp;   // resolves whose step the previous resolve's ballot had shown as the next one not accepted (timing builds)
  long long spec_path[6];  // team evaluations after a failed proof (K winners) | other team evaluations (row not clean,
                           // n_cur > k, a dead current node, too few candidates) | list rebuilds because the list ran
                           // dry | team evaluations that moved data (and rebuilt the list) | extended resolves |
                           // extended scans that found more than SP_XMAX nodes (then a team evaluation)
  long long spec_cyc_team[4];  // of spec_cyc[6], by the first four causes of spec_path (the fourth is part of the first two; timing builds)
  long long spec_cyc_x;    // of spec_cyc[3]: the extended scans and resolves (timing builds)
  long long spec_abort;    // the speculative kernel's watchdog fired (a bug: the plan is reported as failed)
  long long spec_round2;   // resolves that had to look at the second list column
  long long spec_cwait;    // resolves that had to wait for the committer (a pending commit shared their top node)
  long long spec_why[4];   // team evaluations by cause: row not clean | current node dead | candidates ran out | bound test failed
  int32_t masked;          // some node id below N is outside nodesAll (NR_OUTSIDE): such a current node makes a row unclean
};

struct DPool {
  // per partition
  int32_t* rows; int32_t* prev_rows;
  uint32_t* pmeta; uint32_t* prev_meta;
  uint8_t* pflags;
  const int32_t* pweight; const int32_t* name_rank; const int32_t* part_inst;
  unsigned long long* keys; unsigned long long* keys_alt;
  int32_t* order; int32_t* order_alt;
  int32_t* stream; int32_t* ostream;      // step records in / out, [sum PU_i][SLP_i + 8], in step order
  // per node / node id
  const uint8_t* node_removed; const uint8_t* node_added;     // [NU]
  const int32_t* node_weight; const uint8_t* node_has_weight; // [N]
  const int32_t* extra_first; const int32_t* extra_rest;      // [N]
  // tables
  int32_t* counts; int32_t* n2n; const uint32_t* ie_mask;
  // speculative pass: n2n's deviation from the all-sticky hypothesis, the per-step hypothesis counts
  // (qstat[step][4]) and the (top, node) pair sort that produces them
  int32_t* n2n_dev; int32_t* qstat;
  uint8_t* srank;          // [sum PU] per step: 0x80 | ranks of its current nodes when the step was accepted as sticky (sticky_rank.cuh)
  unsigned long long* pair_keys; unsigned long long* pair_keys_alt;
  uint32_t* pair_vals; uint32_t* pair_vals_alt;
  DInst* insts;
};

__host__ __device__ inline uint32_t meta_shape(uint32_t meta, int s) { return (meta >> (2 * s)) & 3u; }
__host__ __device__ inline uint32_t meta_set_shape(uint32_t meta, int s, uint32_t sh) {
  return (meta & ~(3u << (2 * s))) | (sh << (2 * s));
}
