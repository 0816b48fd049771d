/* include/blance_b200.h — C ABI of libblance_b200.so (H100 / sm_90a).
 *
 * This is the drop-in boundary for blance's planner hot path.  The reference
 * (couchbase/blance, pure Go) has no FFI of its own: its boundary is the
 * exported Go API.  A Go host keeps api.go's types and replaces the BODY of
 *
 *     PlanNextMapEx       api.go:147-157  -> planNextMapEx      plan.go:23-58
 *     CalcPartitionMoves  moves.go:41-119
 *
 * with a cgo call into the two entry points below (INTEGRATION.md shows the
 * binding).  Strings never cross: the host interns node / state / partition
 * names to dense int32 ids and passes flat, caller-owned arrays.  All pointers
 * are HOST pointers unless an entry point says otherwise; nothing is retained
 * after a call returns.  Every call returns 0 on success or a negative
 * blance_status; blance_last_error() describes the failure.  There is no CPU
 * fallback: without a usable CUDA device every compute entry point fails.
 *
 * Id spaces
 *   node id      0 .. n_nodes-1 = position in nodesAll (nodePositions, plan.go:72-75);
 *                n_nodes .. n_node_ids-1 = names that appear in rows or in
 *                nodesToRemove / nodesToAdd but not in nodesAll (never candidates);
 *                BLANCE_NO_NODE (-1) = empty slot.
 *   state id     index in sortStateNames(model) order (plan.go:437-447).
 *   partition    index 0 .. n_parts-1 over keys(prevMap) U keys(partitionsToAssign).
 *   rows         int32[n_parts][n_slots]; state s owns slots
 *                [state_slot_off[s], state_slot_off[s+1]), filled from the left in
 *                list order, padded with BLANCE_NO_NODE.  A state's slot range must
 *                hold max(constraints, longest input list of that state).
 *   shape        uint8[n_parts][n_states]: BLANCE_SHAPE_ABSENT (no such key in
 *                NodesByState), _NIL (key present, nil slice), _LIST (non-nil slice).
 *                reflect.DeepEqual (plan.go:38) distinguishes all three.
 */
#ifndef BLANCE_B200_H_
#define BLANCE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BLANCE_NO_NODE (-1)

enum blance_shape { BLANCE_SHAPE_ABSENT = 0, BLANCE_SHAPE_NIL = 1, BLANCE_SHAPE_LIST = 2 };

enum blance_status {
  BLANCE_OK = 0,
  BLANCE_ERR_INVALID_ARG = -1,   /* malformed tables (the reference would panic or misbehave) */
  BLANCE_ERR_UNSUPPORTED = -2,   /* e.g. a CustomNodeSorter (plan.go:580) cannot cross the ABI */
  BLANCE_ERR_CUDA = -3,          /* no device / launch or runtime failure */
  /* -4 is retired (it named a collective library; the data path has no collective) */
  BLANCE_ERR_NOMEM = -5
};

/* NodeScoreBooster (plan.go:693-697) is a Go func value and cannot cross; the
 * only booster in the reference tree is cbgt's (control_test.go:19-26). */
enum blance_booster { BLANCE_BOOSTER_NONE = 0, BLANCE_BOOSTER_CBGT_MAX = 1 };

/* Which kernel runs the sequential greedy chain of a state pass (DESIGN.md section 3).  AUTO picks per
 * pass: the speculative kernel (scout warps + one committing leader) when nearly all rows are clean and many
 * are sticky, the lock-step kernel otherwise.  Results are identical whichever kernel runs. */
enum blance_engine {
  BLANCE_ENGINE_AUTO = 0,
  BLANCE_ENGINE_LOCKSTEP = 1,     /* the lock-step kernel only */
  BLANCE_ENGINE_SEQUENCER = 2     /* round 1's sequencer-window kernel where it applies, else lock-step */
};

typedef struct blance_ctx blance_ctx;   /* owns the device, streams, scratch buffers */

/* device_id < 0: current device.  Replaces nothing in the reference (it has no
 * handle); the Go shim keeps one per process/GPU. */
int blance_ctx_create(blance_ctx** out, int device_id);
/* One context over several GPUs of the node.  blance_plan_next_map_batch() shards its instances over them
 * (instance i -> device_ids[i mod n_devices], one host thread per device; plan instances are independent, so
 * there is no collective in the data path), and the blance_plan_scenarios* calls shard their scenarios the same
 * way; every other entry point runs on device_ids[0].  Errors are reported on this context either way. */
int blance_ctx_create_multi(blance_ctx** out, const int* device_ids, int n_devices);
int blance_ctx_device_count(const blance_ctx* ctx);
void blance_ctx_destroy(blance_ctx* ctx);
const char* blance_last_error(const blance_ctx* ctx);   /* ctx may be NULL: last create error */
int blance_version(void);
/* Number of libblance_b200 kernels launched on this context since it was created
 * (the sort library's own kernels are not counted). */
int64_t blance_ctx_kernel_launches(const blance_ctx* ctx);

/* ---- PlanNextMapEx (api.go:147-157; plan.go:23-331) ------------------------ */
typedef struct blance_plan_in {
  int32_t n_nodes;       /* len(nodesAll) */
  int32_t n_node_ids;    /* >= n_nodes, see "Id spaces" */
  int32_t n_states;      /* len(model) */
  int32_t n_parts;       /* |keys(prevMap) U keys(partitionsToAssign)| */
  int32_t n_slots;       /* = state_slot_off[n_states] */
  int32_t max_iters;     /* MaxIterationsPerPlan, plan.go:21 */
  int32_t top_state;     /* topPriorityStateName, plan.go:126-132 (min priority; first in state order on ties) */
  int32_t booster_kind;  /* enum blance_booster */
  int32_t add_is_nil;        /* nodesToAdd == nil (plan.go:554) */
  int32_t has_part_weights;  /* PartitionWeights != nil (plan.go:105,270,534) */
  int32_t has_node_weights;  /* NodeWeights != nil (plan.go:675) */
  int32_t has_hier_rules;    /* HierarchyRules != nil (plan.go:174) */

  /* per state, [n_states] */
  const int32_t* state_priority;        /* model[s].Priority */
  const int32_t* state_constraints;     /* after ModelStateConstraints override, plan.go:308-319 */
  const int32_t* state_slot_off;        /* [n_states+1] */
  const int32_t* state_stickiness;      /* StateStickiness[s] */
  const uint8_t* state_has_stickiness;  /* key present */

  /* per node id, [n_node_ids] */
  const uint8_t* node_removed;          /* in nodesToRemove (any nonzero value means yes) */
  const uint8_t* node_added;            /* in nodesToAdd */
  /* per node, [n_nodes] */
  const int32_t* node_weight;           /* NodeWeights[n] */
  const uint8_t* node_has_weight;       /* key present */

  /* per partition, [n_parts] */
  const uint8_t* part_in_prev;          /* bit 0: key of prevMap; bit 1 (value 3): that entry also holds state names
                                         * that are not in the model - reflect.DeepEqual (plan.go:38) then never matches
                                         * it, so the first iteration cannot converge */
  const uint8_t* part_in_assign;        /* key of partitionsToAssign */
  const int32_t* part_weight;           /* PartitionWeights[p] */
  const uint8_t* part_has_weight;       /* key present */
  const int32_t* part_name_rank;        /* rank under the name rule of plan.go:519-528,512 (unique) */
  const int32_t* prev_rows;             /* [n_parts][n_slots] prevMap rows (model states only) */
  const uint8_t* prev_shape;            /* [n_parts][n_states] */
  const int32_t* cur_rows;              /* [n_parts][n_slots] partitionsToAssign rows */
  const uint8_t* cur_shape;             /* [n_parts][n_states] */

  /* Weighted node counts contributed by prevMap entries under state names that
   * are NOT in the model (they only feed nodePartitionCounts, plan.go:118-124).
   * first = all of prevMap (iteration 1); rest = only partitions that are not
   * being assigned (iterations >= 2, after plan.go:49-52 replaced the others).
   * [n_nodes] each; NULL = all zero. */
  const int32_t* extra_tot_first;
  const int32_t* extra_tot_rest;

  /* Hierarchy (plan.go:174-226, 703-774), precomputed by the host as bit sets:
   * ie_mask[r][a] = leaves(ancestor(a, include_r)) minus leaves(ancestor(a, exclude_r))
   * for rule r (global index) and anchor a in 0..n_node_ids, where anchor
   * n_node_ids stands for "" (no top-priority node).  Bits 0..n_nodes-1 are node
   * ids; bits n_nodes..n_hier_bits-1 are leaf names outside nodesAll (they only
   * matter for the emptiness test of plan.go:746).  hier_words = ceil(n_hier_bits/32). */
  int32_t n_rules;
  int32_t n_hier_bits;
  const int32_t* rule_off;              /* [n_states+1] rules of state s = [rule_off[s], rule_off[s+1]) */
  const uint32_t* ie_mask;              /* [n_rules][n_node_ids+1][hier_words] */

  int32_t engine;                       /* enum blance_engine; 0 = auto */
} blance_plan_in;

typedef struct blance_plan_out {
  int32_t* next_rows;      /* [n_parts][n_slots]; rows of part_in_assign partitions (others: cur row copy) */
  uint8_t* next_shape;     /* [n_parts][n_states] */
  uint8_t* warn;           /* [n_parts][n_states] 1 = "could not meet constraints" (plan.go:231-234), last iteration only */
  int32_t iters_run;       /* inner plans executed (plan.go:32) */
  int32_t converged;       /* 1 if the last compare of plan.go:36-42 matched */
  int64_t steps;           /* findBestNodes calls executed over all iterations */
  float device_ms;         /* GPU time of the whole call (events on the ctx stream), H2D/D2H included; 0 after
                            * blance_plan_fetch (the resident path has no single call to time) */
  float kernel_ms;         /* GPU time with tables resident (between the copies) */
  float pass_ms;           /* time inside the sequential assign passes only */
  int64_t sticky_steps;    /* of `steps`: accepted scout results / sequencer-window steps (no full evaluation) */
} blance_plan_out;

/* Checks one instance's tables without planning anything and without a device: sizes, pointers and limits (what
 * every planning entry point checks itself) AND the contents - state_slot_off[0] == 0, node ids of both row tables
 * in [-1, n_node_ids), each state's slots filled from the left, shape values, part_name_rank unique and below
 * 2^30, partition weights within the "%10d" rule of plan.go:539, rule_off monotone, and the count bound below.
 * The planning entry points do NOT scan the contents (it would sit in the timed path of every call): a binding that
 * does not trust its own marshalling calls this first.
 *
 * The count bound: the reference counts in 64-bit ints, the device keeps every node's weighted count in int32.
 *     sum_p |w_p| * max(1, n_slots) + max_n max(|extra_tot_first[n]|, |extra_tot_rest[n]|) <= INT32_MAX
 * (w_p = part_weight[p] where has_part_weights and part_has_weight[p], else 1) bounds every such count; an instance
 * above it is BLANCE_ERR_UNSUPPORTED here.  Planning such an instance is undefined: its counts wrap.
 *
 * Returns BLANCE_OK / BLANCE_ERR_INVALID_ARG / BLANCE_ERR_UNSUPPORTED; msg (may be NULL) receives the reason,
 * truncated to msg_cap bytes. */
int blance_plan_in_check(const blance_plan_in* in, char* msg, int32_t msg_cap);

/* Host buffers in, host buffers out.  If prevMap and partitionsToAssign must be
 * mutated as plan.go:49-52 does, the caller copies next_rows back when
 * iters_run >= 2 || !converged. */
int blance_plan_next_map(blance_ctx* ctx, const blance_plan_in* in, blance_plan_out* out);

/* n independent instances (multi-tenant rebalance fan-out); instance i uses
 * in[i] / out[i].  All instances of a device run concurrently (one CTA each per pass); a multi-device
 * context spreads them over its GPUs. */
int blance_plan_next_map_batch(blance_ctx* ctx, int32_t n, const blance_plan_in* in, blance_plan_out* out);

/* ---- what-if scenarios of one cluster ----------------------------------------------------------------------
 * One variant of a base instance: exactly the inputs of PlanNextMapEx that a what-if changes.  Every field is
 * required; the base's own node_removed / node_added / add_is_nil / has_node_weights / node_weight /
 * node_has_weight are ignored by blance_plan_scenarios. */
typedef struct blance_scenario {
  const uint8_t* node_removed;     /* [n_node_ids]  nodesToRemove of this variant */
  const uint8_t* node_added;       /* [n_node_ids]  nodesToAdd of this variant */
  int32_t add_is_nil;              /* nodesToAdd == nil (plan.go:554); 0 or 1 */
  int32_t has_node_weights;        /* NodeWeights != nil (plan.go:675); 0 or 1 */
  const int32_t* node_weight;      /* [n_nodes], read when has_node_weights */
  const uint8_t* node_has_weight;  /* [n_nodes], read when has_node_weights */
} blance_scenario;

/* enum blance_op_kind indexes the second dimension of node_ops */
typedef struct blance_scenario_out {
  int32_t* next_rows;  uint8_t* next_shape;  uint8_t* warn;  /* as blance_plan_out; each may be NULL (not copied) */
  int64_t* node_ops;          /* [n_node_ids][4] ops per node by enum blance_op_kind; may be NULL */
  int64_t* state_node_load;   /* [n_states][n_node_ids]; may be NULL */
  int32_t iters_run, converged;
  int64_t steps, sticky_steps;
  int64_t parts_moved, ops_total, warn_parts;
} blance_scenario_out;

/* Plans n variants of one cluster: scenario i is the plan of `base` with sc[i]'s six node fields substituted,
 * i.e. PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove_i, nodesToAdd_i, model, options with
 * NodeWeights_i) on private copies of the two maps.  out[i].next_rows / next_shape / warn / iters_run /
 * converged / steps equal what blance_plan_next_map returns for that substituted instance, whatever n,
 * max_concurrent, the engine or the number of devices.
 *
 * Summaries (computed on the device; only they, the scalars and the requested row tables are copied out):
 *   node_ops[q][kind], ops_total, parts_moved: for every partition with part_in_assign,
 *     CalcPartitionMoves(states = all model states in state order, beg = its prev_rows row as passed in (a
 *     partition with part_in_prev == 0 starts from an empty row), end = its next row, favor_min_nodes) - the
 *     per-partition call OrchestrateMoves makes (orchestrate.go:273-287).  Each op counts at its node and kind;
 *     ops_total is their sum; parts_moved counts the partitions with at least one op.
 *   state_node_load[s][q]: countStateNodes (plan.go:374-399) over the model states of the final map (prevMap
 *     with every assigned partition replaced by its next row), each entry weighted with the partition's weight
 *     when has_part_weights is set and it has one, else 1.  Removed nodes keep what unassigned partitions hold.
 *   warn_parts: assigned partitions with at least one warning bit.
 *
 * Errors: n <= 0, a NULL sc / out, or a bad scenario (the first one fails the call; the message names its
 * index) is BLANCE_ERR_INVALID_ARG, checked before any device work.  A scenario above the count bound of
 * blance_plan_in_check (on its own partition weights and non-model counts) is BLANCE_ERR_UNSUPPORTED.  Every
 * scenario is checked before ctx is used: with ctx NULL the call returns the first scenario's error, or
 * BLANCE_ERR_INVALID_ARG for the NULL ctx when every scenario passes.  BLANCE_ERR_NOMEM when one scenario does
 * not fit in device memory.
 *
 * Scheduling: the base's partition tables are uploaded once per device and replicated on the device into each
 * scenario of a wave; a wave is one batch through the convergence loop.  max_concurrent > 0 caps the wave size;
 * 0 picks the largest wave that fits the free device memory, and at most sm_count / 2 when the cluster has more
 * than 768 nodes (so every scenario keeps the wide speculative kernel).  A multi-device context sends scenario i
 * to device i mod G, each device with its own copy of the base (DESIGN.md section 8). */
int blance_plan_scenarios(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                          int32_t favor_min_nodes, int32_t max_concurrent, blance_scenario_out* out);

/* Plan options of one scenario (blance_plan_scenarios_ex).  `set` says which groups replace the base's fields;
 * a group whose bit is clear inherits the base and its fields are not read.  Arrays are [n_states] unless noted.
 *
 *   BLANCE_OPT_CONSTRAINTS   ModelStateConstraints (plan.go:308-319): state_constraints.  Every value must fit
 *                            the base's slot range of that state (state_slot_off[s+1] - state_slot_off[s]), so all
 *                            scenarios share the base's row layout.  A binding that lets a scenario raise a
 *                            constraint widens the base's slot ranges up front to the largest constraint of any
 *                            scenario (PlanNextMapScenarios does).
 *   BLANCE_OPT_STICKINESS    StateStickiness: state_stickiness, state_has_stickiness.
 *   BLANCE_OPT_PART_WEIGHTS  PartitionWeights: has_part_weights, and a sparse list of per-partition changes to the
 *                            base's part_weight / part_has_weight: partition ow_part[j] (distinct, in [0, n_parts))
 *                            gets weight ow_weight[j] and presence ow_has[j], each [n_weight_overrides].
 *                            extra_tot_first / extra_tot_rest ([n_nodes], NULL = the base's) replace the counts of
 *                            non-model states (see blance_plan_in): a caller that reweights a partition holding such
 *                            entries must supply them, the device cannot derive them.  The scenario's weights and
 *                            non-model counts must keep the count bound of blance_plan_in_check.
 *   BLANCE_OPT_HIERARCHY     NodeHierarchy and HierarchyRules: has_hier_rules, n_rules, n_hier_bits, rule_off,
 *                            ie_mask, with the meaning they have in blance_plan_in. */
enum blance_scenario_opt_set {
  BLANCE_OPT_CONSTRAINTS = 1,
  BLANCE_OPT_STICKINESS = 2,
  BLANCE_OPT_PART_WEIGHTS = 4,
  BLANCE_OPT_HIERARCHY = 8
};

typedef struct blance_scenario_opts {
  uint32_t set;                         /* OR of enum blance_scenario_opt_set */
  const int32_t* state_constraints;     /* BLANCE_OPT_CONSTRAINTS */
  const int32_t* state_stickiness;      /* BLANCE_OPT_STICKINESS */
  const uint8_t* state_has_stickiness;
  int32_t has_part_weights;             /* BLANCE_OPT_PART_WEIGHTS: 0 or 1 */
  int32_t n_weight_overrides;
  const int32_t* ow_part;
  const int32_t* ow_weight;
  const uint8_t* ow_has;                /* 0 or 1 */
  const int32_t* extra_tot_first;       /* [n_nodes] or NULL */
  const int32_t* extra_tot_rest;        /* [n_nodes] or NULL */
  int32_t has_hier_rules;               /* BLANCE_OPT_HIERARCHY: 0 or 1 */
  int32_t n_rules;
  int32_t n_hier_bits;
  const int32_t* rule_off;              /* [n_states+1] */
  const uint32_t* ie_mask;              /* [n_rules][n_node_ids+1][hier_words] */
} blance_scenario_opts;

/* blance_plan_scenarios with plan options per scenario: scenario i is PlanNextMapEx(prevMap, partitionsToAssign,
 * nodesAll, nodesToRemove_i, nodesToAdd_i, model, options_i), where options_i is the base's options with
 * NodeWeights from sc[i] and the groups of opts[i] replaced.  Everything blance_plan_scenarios promises holds here
 * on the substituted tables (rows, shapes, warnings, iters_run, converged and steps equal blance_plan_next_map;
 * state_node_load weights by the scenario's own partition weights).  opts NULL: no options vary, exactly
 * blance_plan_scenarios.  NodeScoreBooster, MaxIterationsPerPlan, nodesAll and the maps stay shared.
 *
 * Errors, all before any device work, naming the scenario's index: the substituted blance_plan_in fails the
 * checks of blance_plan_next_map (e.g. constraints > 16 or beyond the slot range, rules x constraints > 32, a
 * hierarchy universe above 4096 bits); an unknown bit in `set`; a flag that is neither 0 nor 1; an override index
 * outside [0, n_parts) or listed twice; NULL override arrays (BLANCE_ERR_INVALID_ARG).  An override weight above
 * 999999999 (plan.go:539) or a scenario above the count bound of blance_plan_in_check is BLANCE_ERR_UNSUPPORTED.
 *
 * Scheduling as blance_plan_scenarios; the automatic wave size is priced by the wave's largest scenario (its
 * hierarchy masks), and the overrides are applied on the device after each wave is replicated from the base. */
int blance_plan_scenarios_ex(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                             const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                             blance_scenario_out* out);

/* ---- chains of cluster changes (blance_plan_chains) ---------------------------------------------------------
 * A rolling upgrade, successive failures or repeated rebalances are SEQUENCES of plans, each on the map the one
 * before produced.  Chain i has T = n_stages stages; stage t of chain i is the Go host loop
 *
 *     prev, assign := prevMap, partitionsToAssign              // the base's, never mutated
 *     for t := 0; t < T; t++ {
 *         next, warnings := PlanNextMapEx(prev, assign, nodesAll_t, nodesToRemove_t, nodesToAdd_t, model, options_i_t)
 *         prev = prev with every entry of next replaced         // the stage's FINAL MAP
 *         assign = next
 *     }
 *
 * where nodesAll_t is the base's nodesAll IN BASE ORDER restricted to the ids q < n_nodes with node_in_all[q] = 1
 * (a node that leaves and comes back keeps its position; ids >= n_nodes stay outside nodesAll), nodesToRemove_t /
 * nodesToAdd_t / NodeWeights_t come from the stage's blance_scenario, and options_i_t is the base's options with
 * chain i's opts groups substituted (as blance_plan_scenarios_ex) and NodeWeights_t.  In table terms stage t+1's
 * instance is stage t's with, for every partition with part_in_assign, prev_rows = cur_rows = next_rows,
 * prev_shape = cur_shape = next_shape and part_in_prev = 1 (bit 1 cleared); extra_tot_first = extra_tot_rest (a
 * next row holds model states only: partitionsToAssign may not name other states); and the stage's node fields.
 *
 * out[i * n_stages + t] is a blance_scenario_out with exactly the meaning it has in blance_plan_scenarios, where the
 * "prev row as passed in" is THAT STAGE's prevMap row.  With n_stages = 1 and every node_in_all set, out[i] equals
 * blance_plan_scenarios_ex field for field.  net[i] (net may be NULL; its node_ops may be NULL) holds
 * CalcPartitionMoves over the same states with the same favor_min_nodes from the BASE's prev row (empty when the
 * partition is absent from prevMap) to the LAST stage's next row, for every assigned partition: node_ops, ops_total,
 * parts_moved as in blance_scenario_out.  sum_t out[i * n_stages + t].ops_total - net[i].ops_total is what the
 * sequence moves beyond one direct plan.  Nothing depends on n, max_concurrent, the engine or the number of devices.
 * Schedules, audits and exposures per stage: blance_plan_chains_exposure (below, after blance_plan_scenarios_exposure).
 *
 * Errors, all before any device work: n <= 0, n_stages < 1, a NULL base / stages / out; n_stages > 1 with
 * max_iters < 1 (a stage that plans nothing leaves no next map); a stage that blance_plan_scenarios_ex would reject,
 * a NULL node_in_all, or a node_in_all entry that is neither 0 nor 1 - the message names "chain i, stage t".  With ctx
 * NULL the call returns the first stage's error, or BLANCE_ERR_INVALID_ARG for the NULL ctx.  Scheduling as
 * blance_plan_scenarios (chain i -> device i mod G); a wave's chains run stage by stage in lock step, the map never
 * leaves the device between stages, and the net buffers are priced into the wave size (DESIGN.md section 12).
 * The C++ twin over string maps is PlanNextMapChains (blance_b200/csrc/host_api.hpp). */
typedef struct blance_chain_stage {
  blance_scenario nodes;           /* the stage's nodesToRemove / nodesToAdd / NodeWeights, as a scenario */
  const uint8_t* node_in_all;      /* [n_nodes] 1 = the node is in this stage's nodesAll, 0 = outside */
} blance_chain_stage;

typedef struct blance_chain_out {
  int64_t* node_ops;               /* [n_node_ids][4] by enum blance_op_kind; may be NULL */
  int64_t ops_total, parts_moved;
} blance_chain_out;

int blance_plan_chains(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages,
                       const blance_chain_stage* stages /* [n][n_stages] */, const blance_scenario_opts* opts /* [n] or NULL */,
                       int32_t favor_min_nodes, int32_t max_concurrent, blance_scenario_out* out /* [n][n_stages] */,
                       blance_chain_out* net /* [n] or NULL */);

/* ---- the rebalance schedule of every scenario (blance_plan_scenarios_schedule) --------------------------------
 * Summaries of the lock-step schedule of blance_moves_schedule (rules 1-5 below) of one scenario's moves at one
 * MaxConcurrentPartitionMovesPerNode.  Every array may be NULL (not copied). */
typedef struct blance_scenario_schedule_out {
  int32_t  rounds;           /* R, as blance_schedule_out */
  int64_t  moves_done;       /* ops scheduled */
  int64_t  stuck_parts;      /* partitions whose next move is on a node without a mover */
  int32_t  max_batch;        /* largest batch of one node in one round */
  int32_t* node_rounds;      /* [n_node_ids] rounds in which the node has a batch */
  int32_t* node_last_round;  /* [n_node_ids] 1 + last round with a batch on the node, 0 = none */
  int32_t* part_done_round;  /* [n_parts] 1 + round of the partition's last op; 0 = no ops; -1 = stuck */
} blance_scenario_schedule_out;

/* blance_plan_scenarios_ex, and how long each scenario's rebalance takes.
 *
 * Plans are unchanged: out[i] equals what blance_plan_scenarios_ex returns for the same arguments (rows, shapes,
 * warnings, scalars, node_ops and state_node_load).
 *
 * sched[i * n_move_conc + k] is the lock-step schedule of blance_moves_schedule (rules 1-5 there, unchanged) at
 * MaxConcurrentPartitionMovesPerNode = move_conc[k] (values <= 0 mean 1, orchestrate.go:484-487) of exactly the
 * move lists node_ops counts: for every partition with part_in_assign, CalcPartitionMoves over all model states in
 * state order from its prev row as passed in to its next row (a partition with part_in_prev == 0 starts from an
 * empty row); every other partition has no ops.  In orchestrator terms: OrchestrateMoves(model, {move_conc[k],
 * favor_min_nodes}, nodesAll, begMap = prevMap plus an empty entry for every assigned partition it lacks,
 * endMap = the final map).  So moves_done + the ops left on stuck partitions = ops_total.
 *
 * Partitions are walked in ascending partition index.  node_has_mover ([n_node_ids]) NULL means that exactly the ids
 * < n_nodes (nodesAll) have a mover, as in OrchestrateSchedule, where a node outside nodesAll has none.
 *
 * Summaries, read from the schedule's round_off / sched_op (blance_moves_schedule_fetch):
 *   node_rounds[q]      number of rounds r with an op on node q in round r;
 *   node_last_round[q]  1 + the last such r, 0 if none;
 *   part_done_round[p]  1 + the round of partition p's last op if all its ops were scheduled and it has any; 0 if it
 *                       has no ops; -1 if it is stuck (its next op is on a node without a mover);
 *   rounds, moves_done, stuck_parts and max_batch as blance_schedule_out.
 * Every value equals blance_moves_create (favor_min_nodes, all states visited) + blance_moves_schedule on that
 * scenario's prev and next rows, and none depends on n, max_concurrent, the wave size, the engine, the number of
 * devices or the other values of move_conc.
 *
 * Errors, before any device work, naming the scenario or the index k: everything blance_plan_scenarios_ex rejects;
 * n_move_conc < 1, a NULL move_conc or a NULL sched (BLANCE_ERR_INVALID_ARG); 2^29 or more partitions
 * (BLANCE_ERR_UNSUPPORTED).  BLANCE_ERR_NOMEM when one scenario together with its schedules does not fit in device
 * memory.
 *
 * Scheduling as blance_plan_scenarios_ex.  A scenario's schedule state is priced into the wave size from a bound
 * known before planning (2 x n_slots ops per partition, per count) and allocated with the wave, so the automatic
 * wave never fails for memory because of it; all counts of all scenarios of a wave run in one lock-step sequence
 * on the wave's device (DESIGN.md section 10). */
int blance_plan_scenarios_schedule(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                   const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                   int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                   blance_scenario_out* out, blance_scenario_schedule_out* sched);

/* Device-resident variant used by benchmarks and by callers that chain plans:
 * uploads `in` once and returns a handle; blance_plan_run() replays the whole
 * plan on the resident tables (inputs are restored on device before each run);
 * blance_plan_fetch() copies the result out. */
typedef struct blance_plan blance_plan;
int blance_plan_upload(blance_ctx* ctx, const blance_plan_in* in, blance_plan** plan);
int blance_plan_run(blance_ctx* ctx, blance_plan* plan);
int blance_plan_fetch(blance_ctx* ctx, blance_plan* plan, blance_plan_out* out);
void blance_plan_free(blance_ctx* ctx, blance_plan* plan);
/* Device times of the last blance_plan_run (CUDA events on the ctx stream): the whole
 * run, the part spent inside the sequential assign-pass kernels, and how many of
 * those were launched. */
int blance_plan_timing(const blance_plan* plan, float* kernel_ms, float* pass_ms, int32_t* pass_launches);

/* ---- auditing a partition map (blance_map_audit, blance_plan_audit, blance_plan_scenarios_audit) ---------------
 * The planner reports one kind of problem, "could not meet constraints" (plan.go:228-235).  It is silent when a
 * hierarchy rule's candidate set is empty and findBestNodes falls back to the flat best node (plan.go:214-220): a
 * replica lands in its primary's rack and nothing says so.  An audit counts, over a finished map, the unmet
 * constraints, the placements that miss a hierarchy rule and what each node or fault domain holds.  It audits the map
 * against the rule as the planner applies it to a finished row; it does NOT replay the pass (the planner anchored
 * the top state's own pass on the OLD primary, and carried one rule's picks into the next rule's prefix).
 *
 * Inputs: one map (rows + shapes in the layout of "Id spaces"), the model (n_states, state_slot_off,
 * state_constraints, top_state), optionally the hierarchy rules (has_hier_rules, n_rules, n_hier_bits, rule_off,
 * ie_mask) and optionally a fault-domain forest.  Only model states count.  For partition p, L_s is its list of
 * state s: it HAS a list when shape[p][s] != BLANCE_SHAPE_ABSENT, and len(L_s) is the number of nodes before the
 * first BLANCE_NO_NODE of the state's slot range (0 for a nil slice, whatever its slots hold).  Node ids must lie in
 * [-1, n_node_ids) (blance_plan_in_check scans for that; the audit does not): an id outside that range counts
 * towards len(L_s) but is no copy, never complies, and as a prefix element stands for "".  h is the first node of its list of
 * top_state, or the "" anchor (id n_node_ids) when that list is absent or empty (plan.go:134-138).  A copy is one
 * (state, position) entry of any list of p.
 *
 * Constraints (states with state_constraints[s] > 0, partitions that have a list for s; the static form of
 * plan.go:228, which also sees partitions that were not assigned - `warn` never does):
 *   short_slots[s] = sum over p of max(0, state_constraints[s] - len(L_s));  short_parts = partitions with any
 *   shortfall;  over_slots[s] = sum over p of max(0, len(L_s) - state_constraints[s]).
 *
 * Hierarchy rules (has_hier_rules; states with rules and state_constraints[s] > 0).  Position j of L_s is TESTED
 * when j < min(len(L_s), state_constraints[s]), except position 0 of top_state (it is the anchor).  For rule r of
 * state s (global index rule_off[s] <= r < rule_off[s+1]) the node x = L_s[j] COMPLIES iff x < n_nodes (the planner
 * picks from nodesNext only, plan.go:193-194) and bit x is set in
 *   includeExcludeNodesIntersect([a] + L_s[0..j-1], r.IncludeLevel, r.ExcludeLevel)      (plan.go:738-753)
 * read literally over the bit sets ie_mask[r][.]: rv starts empty; for every node y of the list in order, rv becomes
 * ie_mask[r][y] when rv is empty (the replace-on-empty step of plan.go:746-749, over all n_hier_bits bits), else
 * rv AND ie_mask[r][y].  The anchor a is h; when h is "" and j > 0 it is L_s[0] (plan.go:178-181); when h is "" and
 * j = 0 it is "" itself.
 *   rule_tested[r] = tested (partition, position) pairs;  rule_miss[r] = those that do not comply;
 *   rule_miss_parts = partitions with at least one miss.
 *
 * Fault domains.  domain_parent[n_node_ids + n_domains]: vertices 0 .. n_node_ids-1 are the node ids, the rest are
 * inner vertices (racks, zones); domain_parent[v] is v's parent vertex or -1 for a root; every vertex is at most 16
 * edges below its root.  NULL (with n_domains = 0) means every node is its own domain.  A vertex contains itself.
 *   dom_copies[v] = copies on nodes under v;
 *   dom_top[v]    = partitions whose h lies under v (they need a promotion if v fails);
 *   dom_all[v]    = partitions with at least one copy whose EVERY copy lies under v (they are lost if v fails): per
 *                   partition the deepest common ancestor of its copies and every vertex from there to the root.
 *   no_top_parts  = partitions whose h is "".
 *
 * Failover spread (BLANCE_AUDIT_N2N).  n2n[a][b] (a, b < n_nodes) = number of copies on b of partitions with h = a,
 * b != a: the final-map form of the nodeToNodeCounts the score spreads (plan.go:238-245).  n2n_max is its largest
 * entry and (n2n_max_a, n2n_max_b) the lowest (a, b) that holds it - the node that takes the most promotions when a
 * fails; (-1, -1) when the matrix is all zero.  Without the flag no matrix exists on the device and the three
 * scalars are -1.
 *
 * part_flags[p]: bit 0 = short, bit 1 = rule miss, bit 2 = h is "".
 * All counts are unweighted; none depends on thread order, the wave size, the engine or the number of devices. */
enum blance_audit_flags { BLANCE_AUDIT_N2N = 1 };

typedef struct blance_audit_opts {
  uint32_t flags;                 /* OR of enum blance_audit_flags */
  int32_t n_domains;              /* inner vertices of the forest; 0 when domain_parent is NULL */
  const int32_t* domain_parent;   /* [n_node_ids + n_domains] or NULL */
} blance_audit_opts;

/* Every array may be NULL (not copied).  V = n_node_ids + n_domains; n_rules is the audited instance's own (0
 * without has_hier_rules). */
typedef struct blance_audit_out {
  int64_t* short_slots;           /* [n_states] */
  int64_t* over_slots;            /* [n_states] */
  int64_t* rule_miss;             /* [n_rules] */
  int64_t* rule_tested;           /* [n_rules] */
  int64_t* dom_top;               /* [V] */
  int64_t* dom_all;               /* [V] */
  int64_t* dom_copies;            /* [V] */
  int32_t* n2n;                   /* [n_nodes][n_nodes], BLANCE_AUDIT_N2N only */
  uint8_t* part_flags;            /* [n_parts] */
  int64_t short_parts, rule_miss_parts, no_top_parts;
  int32_t n2n_max, n2n_max_a, n2n_max_b;
  float kernel_ms;                /* GPU time of the audit kernels (events around them); in a scenario wave, of the whole
                                   * wave's audits, the same value in each of its scenarios */
} blance_audit_out;

/* Audits the map (rows [n_parts][n_slots], shape [n_parts][n_states]) against `model`, of which only the sizes, the
 * state tables state_slot_off / state_constraints / top_state and the hierarchy fields are read; its own row and
 * partition tables are ignored and may be NULL.  opts NULL = no flags, nodes only.
 * Errors, all before any device work: a NULL model, out, rows or shape (with partitions and slots / states to
 * read); sizes beyond the limits of blance_plan_next_map (8 states, 32 slots, 4096 hierarchy bits ->
 * BLANCE_ERR_UNSUPPORTED), more than 256 rules (BLANCE_ERR_UNSUPPORTED); an unknown flag; n_domains < 0 or without
 * domain_parent; a domain_parent entry outside [-1, V), a cycle or a vertex more than 16 edges below its root
 * (BLANCE_ERR_INVALID_ARG).  Then, without a usable device, BLANCE_ERR_CUDA (also when ctx is NULL because none
 * could be created). */
int blance_map_audit(blance_ctx* ctx, const blance_plan_in* model, const int32_t* rows, const uint8_t* shape,
                     const blance_audit_opts* opts, blance_audit_out* out);

/* The same audit of a resident plan's map as it stands on the device - the result of the last blance_plan_run, the
 * uploaded partitionsToAssign rows before any run - under the plan's own model and hierarchy, with no copy of the
 * rows: equal to blance_map_audit on the rows and shapes blance_plan_fetch returns. */
int blance_plan_audit(blance_ctx* ctx, blance_plan* plan, const blance_audit_opts* opts, blance_audit_out* out);

/* blance_plan_scenarios_schedule, and an audit of every scenario's final map.
 *
 * out and sched equal what blance_plan_scenarios_schedule returns for the same arguments.  n_move_conc = 0 with a
 * NULL move_conc and sched asks for no schedule (out then equals blance_plan_scenarios_ex).
 * audit[i] (n entries) equals blance_map_audit of scenario i's FINAL MAP - prevMap with every assigned partition
 * replaced by its next row, the map state_node_load is defined over; a partition in neither map has no lists -
 * under scenario i's own constraints and hierarchy (blance_scenario_opts) and the shared `aopts`.  The audit runs
 * inside the wave, next to the summaries and before anything is copied out; its buffers are priced into the wave
 * size (a few KB per scenario, plus n_nodes x n_nodes x 4 bytes with BLANCE_AUDIT_N2N).
 * Errors as blance_plan_scenarios_schedule and blance_map_audit, plus a NULL audit, all before any device work.
 * blance_plan_scenarios_exposure (below, after blance_moves_exposure) adds the exposure of every scenario's schedule. */
int blance_plan_scenarios_audit(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                blance_scenario_out* out, blance_scenario_schedule_out* sched,
                                const blance_audit_opts* aopts, blance_audit_out* audit);

/* ---- CalcPartitionMoves (moves.go:41-119), vectorised over partitions ------- */
enum blance_op_kind { BLANCE_OP_ADD = 0, BLANCE_OP_DEL = 1, BLANCE_OP_PROMOTE = 2, BLANCE_OP_DEMOTE = 3 };
#define BLANCE_OP_STATE_NONE 0xFF   /* the "" state of a del op (moves.go:87) */

/* beg_rows/end_rows: [n_parts][n_slots] with the slot layout of state_slot_off
 * ([n_states+1]).  Only the first n_visit_states states are walked as `states`
 * (moves.go:66,92); the remaining ones still count for adds/dels (moves.go:60-64).
 * Outputs: op_* are [n_parts][max_ops] (max_ops >= 2*n_slots is always enough),
 * op_count[n_parts] = number of ops of each partition, in the reference's order. */
int blance_calc_partition_moves(blance_ctx* ctx, int32_t n_parts, int32_t n_states, int32_t n_visit_states,
                                const int32_t* state_slot_off, const int32_t* beg_rows,
                                const int32_t* end_rows, int32_t favor_min_nodes, int32_t max_ops,
                                int32_t* op_node, uint8_t* op_state, uint8_t* op_kind, int32_t* op_count);

/* ---- move lists for the orchestrator (orchestrate.go:273-287, 749-763, 177-186) ----------------------------
 * OrchestrateMoves seeds one NextMoves{Moves: CalcPartitionMoves(...)} per partition (orchestrate.go:273-287),
 * then repeatedly rebuilds "which partitions have their NEXT move on node n" by scanning every partition
 * (findAvailableMovesUnlocked, orchestrate.go:749-763) and lets the FindMoveFunc pick one per node
 * (LowestWeightPartitionMoveForNode, orchestrate.go:177-186: the lowest MoveOpWeight wins).  A blance_moves
 * handle keeps all move lists on the device in CSR form; blance_moves_available() answers one round of the
 * scan for a vector of cursors.
 *   Order: the reference appends in Go map order (random); here every per-node list is in ascending partition
 *   index, and ties of the lowest weight go to the lowest partition index. */
typedef struct blance_moves blance_moves;

/* beg_rows / end_rows / state_slot_off / n_visit_states / favor_min_nodes as in blance_calc_partition_moves.
 * n_node_ids bounds the node ids that occur in the rows.  *total_ops receives the number of ops of all
 * partitions together (the size of the op_* arrays blance_moves_fetch fills).  The handle also keeps the beg rows and
 * the slot layout on the device, for blance_moves_exposure. */
int blance_moves_create(blance_ctx* ctx, int32_t n_parts, int32_t n_states, int32_t n_visit_states,
                        const int32_t* state_slot_off, const int32_t* beg_rows, const int32_t* end_rows,
                        int32_t favor_min_nodes, int32_t n_node_ids, blance_moves** out, int64_t* total_ops);
/* CSR copy-out: op_off[n_parts+1]; op_node / op_state / op_kind [total_ops], partition p owns [op_off[p], op_off[p+1]). */
int blance_moves_fetch(blance_ctx* ctx, blance_moves* moves, int64_t* op_off, int32_t* op_node, uint8_t* op_state,
                       uint8_t* op_kind);
/* One round of findAvailableMovesUnlocked for cursors next[n_parts] (NextMoves.Next): node_off[n_node_ids+1] and
 * node_parts[<= n_parts] list, per node, the partitions whose next move is on it (ascending partition index);
 * best_part[n_node_ids] is the FindMoveFunc's pick with MoveOpWeight {promote 1, demote 2, add 3, del 4}, or -1
 * when the node has no available move.  Any output pointer may be NULL. */
int blance_moves_available(blance_ctx* ctx, blance_moves* moves, const int32_t* next, int32_t* node_off,
                           int32_t* node_parts, int32_t* best_part);

/* ---- the orchestrator's whole schedule (orchestrate.go:482-504, 509-591, 749-763, 177-186) -----------------
 * The Go orchestrator is goroutines and callbacks; Go's map order and its select between broadcastStopCh and
 * nextDoneCh make every run's interleaving nondeterministic.  blance_moves_schedule() does not reproduce one run:
 * it computes the schedule of a LOCK-STEP MODEL of the same statements:
 *   1. every cursor starts at 0 (NextMoves.Next);
 *   2. a round begins with findAvailableMovesUnlocked: every partition with next < len(moves) is appended to the
 *      list of moves[next].Node, walking partitions in ASCENDING INDEX (the order of blance_moves_available);
 *   3. for every node with a non-empty list, in ascending node id, filterNextPlausibleMovesForNode runs as
 *      orchestrate.go:482-504: count = max(1, max_concurrent_per_node), capped at the list length; each pick is
 *      LowestWeightPartitionMoveForNode - the FIRST index of minimal MoveOpWeight {promote 1, demote 2, add 3,
 *      del 4} over the array as it stands - and the picked entry is replaced by the last one, the array shrinking
 *      by one.  The picks, in pick order, are the node's batch (one AssignPartitionsFunc call);
 *   4. every batch of the round completes before the next round (no errors, pause or stop); each picked
 *      partition's cursor advances by one;
 *   5. a move on a node without a mover (node_has_mover[n] == 0, or a node id outside [0, n_node_ids)) is never
 *      picked: the reference would send on a nil channel and hang.  That partition never advances; the schedule
 *      ends when no pickable move is left and stuck_parts counts the partitions left behind.
 * FindMoveFunc is always LowestWeightPartitionMoveForNode and MoveOpWeight keeps its default values: Go func values
 * and package variables cannot cross the ABI (the same policy as NodeScoreBooster).
 *
 * Result: R rounds; round_off[R+1] (int64, round_off[0] = 0) and sched_op[moves_done]: global op indices into the
 * CSR arrays of blance_moves_fetch, ordered by round, then node id, then pick order.  Round r's ops are
 * sched_op[round_off[r] .. round_off[r+1]); node, state and kind of each come from blance_moves_fetch.
 *
 * blance_moves_schedule computes the schedule on the device in one call (the host waits for the device once per
 * 64 rounds) and keeps it in the handle until the next blance_moves_schedule or blance_moves_free;
 * blance_moves_schedule_fetch copies it out (round_off: R+1 entries, sched_op: moves_done entries; either may be
 * NULL).  Scratch is allocated and freed inside the call; blance_moves_available is not affected.  Repeated calls
 * give identical results.  node_has_mover: [n_node_ids], NULL = every id has a mover.  Errors: NULL ctx, handle or
 * out (BLANCE_ERR_INVALID_ARG); a handle with 2^29 or more partitions (BLANCE_ERR_UNSUPPORTED, before any device
 * work); fetch before any schedule (BLANCE_ERR_INVALID_ARG). */
typedef struct blance_schedule_out {
  int32_t rounds;        /* R */
  int64_t moves_done;    /* ops scheduled = length of sched_op = round_off[R] */
  int64_t stuck_parts;   /* partitions whose next move is on a node without a mover */
  int32_t max_batch;     /* largest batch of one node in one round */
  float device_ms;       /* CUDA events around the whole call */
} blance_schedule_out;

int blance_moves_schedule(blance_ctx* ctx, blance_moves* moves, int32_t max_concurrent_per_node,
                          const uint8_t* node_has_mover, blance_schedule_out* out);
int blance_moves_schedule_fetch(blance_ctx* ctx, blance_moves* moves, int64_t* round_off, int64_t* sched_op);

/* ---- the exposure of a rebalance (blance_moves_exposure) ---------------------------------------------------
 * Is the data safe while a rebalance runs?  favorMinNodes (moves.go:35-40) trades "the least number of nodes at any
 * time" against "availability across multiple nodes during moves": a primary moving from a to b is del a, add b
 * (no copy in between) with favor_min_nodes, add b, del a (two primaries in between) without.  The exposure counts
 * that cost over the maps a rebalance passes through under the handle's LAST blance_moves_schedule (R rounds,
 * round_off, sched_op), on the device, without copying the schedule or any map out.
 *
 * Maps.  For t = 0 .. R, M_t is the map after t completed rounds.  M_0 is the handle's beg rows.  Partition p's ops
 * are applied in CSR order; op k is applied at the end of the round rho_k that scheduled it, so it is in M_t for
 * t > rho_k.  An op that was never scheduled (a stuck partition's remaining ops) is never applied.  Applying op
 * (node n, state s, kind) is what the reference's test app does with an AssignPartitionsFunc call
 * (orchestrate_test.go:137-157; orchestrate.go:143-152): every entry of n leaves the partition's lists and, unless the
 * kind is BLANCE_OP_DEL (state ""), one entry (n, s) is added.
 * Entries.  A partition's entries are its (state, position) entries as the move lists read a row: the slots of a
 * state before its first BLANCE_NO_NODE.  A node listed twice in a beg row counts twice until its op.  CalcPartitionMoves'
 * seen rule (moves.go:51-58) gives a node at most one op per partition, so when its op runs a node's entries are
 * exactly its beg entries.  rho_k strictly increases along a partition's ops, so each of its intermediate states is
 * some M_t: per-partition results are exact over the op sequence; only the coincidence across partitions depends on
 * the lock-step model.
 *
 * For partition p in M_t with c_s entries of state s and C = sum_s c_s, metric m (enum blance_expo_metric) counts:
 *   NO_TOP     top_state >= 0 and c_top = 0 (no primary)
 *   MULTI_TOP  top_state >= 0, state_constraints[top] > 0 and c_top > state_constraints[top]
 *   SHORT      some s has state_constraints[s] > 0 and c_s < state_constraints[s]
 *   ONE_COPY   C = 1
 *   NO_COPY    C = 0
 *   COPIES     (not a count of partitions) sum_p C
 *
 * Inputs: state_constraints[n_states] (0 = not constrained; use 0 for states outside the model), top_state (-1 for
 * none), and optionally a fault-domain forest with the meaning and checks of blance_audit_opts (V = n_node_ids +
 * n_domains; NULL: every node is its own domain).
 * Outputs (every array may be NULL):
 *   rounds                     R, echoed
 *   series[m][R + 1]           metric m on M_t
 *   peak[m], peak_round[m]     its largest value and the smallest t that reaches it;  area[m] = sum_t series[m][t]
 *   dom_peak[V]                max over t of the partitions with C >= 1 whose every entry lies on a node under v in M_t
 *                              (an entry on an id outside [0, n_node_ids) lies under no vertex); without a forest,
 *                              dom_peak[q] is the most partitions node q alone held at any moment of the rebalance
 *   dom_peak_round[V]          the smallest t at which dom_peak[v] is reached
 *   part_min_copies[n_parts]   min over t of C;   part_no_top[n_parts]  number of t in 0 .. R at which NO_TOP holds
 *   part_flags[n_parts]        bit m: the partition is counted in metric m at some t (bit COPIES: C > 0 at some t)
 *   kernel_ms                  GPU time of the exposure (events around its device work)
 * Every value equals a literal replay of the schedule; nothing depends on thread order.
 *
 * Errors, before any device work: a NULL ctx, moves, in or out, a handle without a schedule, NULL constraints with
 * states, a negative constraint, top_state outside [-1, n_states), a bad forest (as blance_map_audit)
 * (BLANCE_ERR_INVALID_ARG); more than 8 states or 32 slots, or dom_peak / dom_peak_round asked for with
 * 2 x 17 x moves_done >= 2^31 (BLANCE_ERR_UNSUPPORTED).  The device work is bounded by the handle's sizes plus, with
 * dom_peak, an event buffer of at most 2 x 17 entries per scheduled op (DESIGN.md section 13); BLANCE_ERR_NOMEM when
 * that does not fit.  The C++ twin over string maps is OrchestrateExposure (blance_b200/csrc/host_api.hpp). */
enum blance_expo_metric {
  BLANCE_EXPO_NO_TOP = 0, BLANCE_EXPO_MULTI_TOP = 1, BLANCE_EXPO_SHORT = 2, BLANCE_EXPO_ONE_COPY = 3,
  BLANCE_EXPO_NO_COPY = 4, BLANCE_EXPO_COPIES = 5, BLANCE_EXPO_N = 6
};

typedef struct blance_exposure_in {
  const int32_t* state_constraints;   /* [n_states] of the handle */
  int32_t top_state;                  /* -1: none */
  int32_t n_domains;                  /* inner vertices of the forest; 0 when domain_parent is NULL */
  const int32_t* domain_parent;       /* [n_node_ids + n_domains] or NULL */
} blance_exposure_in;

typedef struct blance_exposure_out {
  int32_t rounds;
  int64_t* series;                    /* [BLANCE_EXPO_N][rounds + 1] */
  int64_t peak[BLANCE_EXPO_N];
  int32_t peak_round[BLANCE_EXPO_N];
  int64_t area[BLANCE_EXPO_N];
  int64_t* dom_peak;                  /* [V] */
  int32_t* dom_peak_round;            /* [V] */
  int32_t* part_min_copies;           /* [n_parts] */
  int32_t* part_no_top;               /* [n_parts] */
  uint8_t* part_flags;                /* [n_parts] */
  float kernel_ms;
} blance_exposure_out;

int blance_moves_exposure(blance_ctx* ctx, blance_moves* moves, const blance_exposure_in* in, blance_exposure_out* out);

/* ---- each node's load while a rebalance runs (blance_moves_load) ---------------------------------------------
 * Does a node run out of room while the rebalance runs?  Without favor_min_nodes every move adds the new copy before
 * it deletes the old one (moves.go:35-40), so a node that gains copies early and loses its own late holds more, at
 * some round in between, than both its start and its end load.  The load counts that over the maps a rebalance passes
 * through under the handle's LAST blance_moves_schedule, on the device, without copying the schedule or any map out.
 *
 * Maps and entries are exactly those of blance_moves_exposure: M_0 .. M_R, M_0 the handle's beg rows, op k applied
 * at the end of its round rho_k, an op that was never scheduled never applied.
 * Weight.  Partition p weighs w_p: part_weight[p] when it has one, else 1 (the rule of countStateNodes,
 * plan.go:374-399, and of state_node_load).  part_weight NULL: every partition weighs 1; part_has_weight NULL with a
 * part_weight: every partition has its weight.
 * Load.  load_t[s][q] is the sum of w_p over the entries (q, s) of M_t; row s = n_states is the sum over all states.
 * An entry on an id outside [0, n_node_ids) counts nowhere.
 * Outputs (every array may be NULL; arrays are [n_states + 1][n_node_ids]):
 *   rounds                     R, echoed
 *   node_beg, node_end         the load on M_0 and on M_R (node_end is not the end rows' load when partitions are stuck)
 *   node_peak                  max over t of load_t
 *   node_peak_round            the smallest t that reaches it
 *   over_max, over_node        the largest node_peak[S][q] - max(node_beg[S][q], node_end[S][q]) and the lowest q
 *                              that reaches it (over_node = -1 without node ids): how far the busiest node overshoots
 *                              both ends of the rebalance
 *   kernel_ms                  time of the load on the stream: events around its device work, which also span the
 *                              host's two waits for the stream (the event count, then the merged runs) and the
 *                              allocation of the event buffer between them
 * Every value equals a literal replay of the schedule; nothing depends on thread order.  No output is sized by
 * nodes x rounds: there is no per-node series.
 *
 * Bounds.  On any M_t node q holds, for partition p, either its beg entries or at most one entry, so its load is at
 * most sum_p w_p x max(n_slots, 1); the call refuses that reaching 2^31, and below it every load is exact.
 * Errors, before any device work: a NULL ctx, moves, in or out, a handle without a schedule, a weight below 0 or
 * above 999999999 (BLANCE_ERR_INVALID_ARG); more than 8 states or 32 slots, the load bound above, (n_slots + 1) x
 * moves_done >= 2^31 (each scheduled op emits at most n_slots + 1 load changes) or (n_states + 1) x n_node_ids >= 2^32
 * (BLANCE_ERR_UNSUPPORTED).  The device work is bounded by the handle's sizes plus an event buffer sized exactly by a
 * counting pass (DESIGN.md section 18); BLANCE_ERR_NOMEM names the load when that does not fit. */
typedef struct blance_load_in {
  const int32_t* part_weight;         /* [n_parts] or NULL */
  const uint8_t* part_has_weight;     /* [n_parts] or NULL */
} blance_load_in;

typedef struct blance_load_out {
  int32_t rounds;
  int64_t* node_beg;                  /* [n_states + 1][n_node_ids] */
  int64_t* node_end;                  /* [n_states + 1][n_node_ids] */
  int64_t* node_peak;                 /* [n_states + 1][n_node_ids] */
  int32_t* node_peak_round;           /* [n_states + 1][n_node_ids] */
  int64_t over_max;
  int32_t over_node;
  float kernel_ms;
} blance_load_out;

int blance_moves_load(blance_ctx* ctx, blance_moves* moves, const blance_load_in* in, blance_load_out* out);

/* ---- each node's load while every scenario's rebalance runs (blance_plan_scenarios_load) -----------------------
 * blance_plan_scenarios_exposure with the exposure optional (expo NULL: none; eopts and series_cap are then only
 * checked), and the node load of every (scenario, count) pair's schedule inside the wave.  out, sched, audit and expo
 * equal what blance_plan_scenarios_exposure returns for the same arguments (with expo NULL: blance_plan_scenarios_audit,
 * or blance_plan_scenarios_schedule with audit NULL too).
 *
 * load[i * n_move_conc + k] equals blance_moves_load on the handle of scenario i's rebalance at move_conc[k], the
 * handle and its schedule as blance_plan_scenarios_exposure defines them for expo, with scenario i's own partition
 * weights (its BLANCE_OPT_PART_WEIGHTS overrides applied; weight 1 where has_part_weights is 0 or a partition has
 * none): the rule of state_node_load, so with no stuck partition node_end's state rows equal out[i].state_node_load.
 * A partition in neither map is no partition of begMap and counts nowhere.  The count bound every scenario passes
 * (sum of |weight| x max(n_slots, 1) < 2^31) bounds every node's load on every map, so the loads are exact; a weight
 * may be negative where the planner allows one.  kernel_ms is the wave's load time (as blance_moves_load measures it,
 * over all its members), the same value in each of its members.  No value depends on n, max_concurrent, the wave
 * size, the engine, the number of devices or the other move_conc.
 *
 * Errors, all before any device work: everything blance_plan_scenarios_exposure rejects except a NULL expo; a NULL
 * load (BLANCE_ERR_INVALID_ARG); (n_slots + 1) x 2 x n_slots x n_parts >= 2^31 or (n_states + 1) x n_node_ids >= 2^32
 * (BLANCE_ERR_UNSUPPORTED, the static forms of blance_moves_load's event and key bounds).  The per-instance outputs
 * (36 bytes per (state, node) and 16 per partition) are priced into the wave size; the event buffers are allocated
 * after the schedules, exactly sized for the wave's instance with the most events, and BLANCE_ERR_NOMEM names the
 * load when they do not fit (DESIGN.md section 18). */
int blance_plan_scenarios_load(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                               const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                               int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                               blance_scenario_out* out, blance_scenario_schedule_out* sched,
                               const blance_audit_opts* aopts, blance_audit_out* audit /* [n] or NULL */,
                               const blance_audit_opts* eopts, int32_t series_cap,
                               blance_exposure_out* expo /* [n][n_move_conc] or NULL */,
                               blance_load_out* load /* [n][n_move_conc] */);

/* ---- the exposure of every scenario's rebalance (blance_plan_scenarios_exposure) ----------------------------
 * blance_plan_scenarios_audit, and the exposure of every (scenario, count) pair's schedule, inside the wave.
 *
 * Arguments up to audit mean what they mean in blance_plan_scenarios_audit, except that audit may be NULL (no audit;
 * aopts is then not read).  out, sched and audit equal what blance_plan_scenarios_audit returns for the same
 * arguments; with audit NULL, out and sched equal blance_plan_scenarios_schedule.
 *
 * expo[i * n_move_conc + k] equals blance_moves_exposure on the handle of scenario i's rebalance at move_conc[k]:
 *   partitions   those of its begMap - part_in_prev || part_in_assign - in ascending partition index;
 *   beg row      the prev row as passed in (model states only; an assigned partition absent from prevMap starts
 *                from an empty row); end row: the next row for an assigned partition, the prev row otherwise;
 *   handle       favor_min_nodes, all states visited, scheduled at move_conc[k] with node_has_mover (the schedule
 *                sched[i * n_move_conc + k] reports);
 *   exposure_in  scenario i's own state_constraints (BLANCE_OPT_CONSTRAINTS applies), the base's top_state and the
 *                forest of eopts (flags must be 0; NULL = every node its own domain).
 * The per-partition arrays are [n_parts] over all partitions: a partition in neither map is no partition of begMap,
 * counts in no metric and gets part_min_copies = -1, part_no_top = 0 and part_flags = 0.
 * series is [BLANCE_EXPO_N][series_cap]: the first min(R + 1, series_cap) values of each metric (R = rounds, so a
 * caller sees when the series was cut; R is not known before planning).  peak, peak_round and area always cover all
 * R + 1 maps.  series_cap = 0 or a NULL series asks for none.  dom_peak / dom_peak_round are computed only when some
 * expo[] asks for one of them.  kernel_ms is the wave's exposure time, the same value in each of its members.
 * No value depends on n, max_concurrent, the wave size, the engine, the number of devices or the other move_conc.
 *
 * Errors, all before any device work, naming the scenario or k: everything blance_plan_scenarios_audit rejects;
 * n_move_conc < 1, a NULL expo, series_cap < 0, eopts with flags set or a bad forest (BLANCE_ERR_INVALID_ARG);
 * dom_peak or dom_peak_round asked for with 2 x 17 x 2 x n_slots x n_parts >= 2^31 (BLANCE_ERR_UNSUPPORTED, the
 * static form of blance_moves_exposure's bound).  The op states and rounds and the outputs asked for are priced
 * into the wave size; the per-round arrays (48 bytes per round and instance) and the fault-domain events are
 * allocated after the schedule, exactly sized, and BLANCE_ERR_NOMEM names the exposure when they do not fit
 * (DESIGN.md section 14). */
int blance_plan_scenarios_exposure(blance_ctx* ctx, const blance_plan_in* base, int32_t n, const blance_scenario* sc,
                                   const blance_scenario_opts* opts, int32_t favor_min_nodes, int32_t max_concurrent,
                                   int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                   blance_scenario_out* out, blance_scenario_schedule_out* sched,
                                   const blance_audit_opts* aopts, blance_audit_out* audit /* [n] or NULL */,
                                   const blance_audit_opts* eopts /* forest only, flags must be 0; NULL = nodes only */,
                                   int32_t series_cap, blance_exposure_out* expo /* [n][n_move_conc] */);

/* ---- schedules, audits and exposures of every chain stage (blance_plan_chains_exposure) ---------------------
 * blance_plan_chains, and for every stage of every chain what blance_plan_scenarios_exposure gives for one scenario:
 * how many rounds each step of a rolling upgrade takes, whether a step leaves partitions without a primary or on one
 * node, and whether the map after each step meets its constraints and hierarchy rules.  T = n_stages, nc = n_move_conc.
 *
 * Plans are unchanged: out and net equal blance_plan_chains for the same arguments, byte for byte.
 *
 * Per stage.  sched[(i * T + t) * nc + k], audit[i * T + t] and expo[(i * T + t) * nc + k] are what
 * blance_plan_scenarios_exposure defines for one scenario, where "prevMap" is STAGE t's prevMap: begMap = stage t's
 * prevMap plus an empty entry for every assigned partition it lacks, the end map is stage t's final map, the
 * constraints and hierarchy are chain i's own (opts[i]), the top state the base's and the forest that of eopts.  With
 * T = 1 and every node_in_all set the result equals blance_plan_scenarios_exposure field for field.
 *
 * Net.  net_sched[i * nc + k] and net_expo[i * nc + k] are the schedule and exposure of the direct rebalance from the
 * BASE's prevMap to the last stage's final map - the moves net[i] counts: the chain against one direct jump.
 *
 * Movers.  One node_has_mover [n_node_ids] serves every stage and the net rebalance; NULL means the ids < n_nodes,
 * the universe, as OrchestrateSchedule has them.  A stage's ops only touch nodes in that stage's nodesAll when every
 * node that leaves nodesAll was removed in an earlier stage (removal strips a node from every assigned row).  The
 * string twin's default NodesAll rule guarantees that, and the result then equals OrchestrateSchedule(nodesAll_t, ...).
 * Per-chain, per-stage mover sets are not supported.
 *
 * Span.  span[i * nc + k] folds chain i's stages at move_conc[k] into one record, on the device.  R_t is stage t's
 * rounds and G_t = sum_{u < t} R_u the global round at which stage t starts.  Every span array may be NULL; nothing in
 * the span depends on whether the per-stage arrays were asked for (they may all be NULL while the span is complete).
 * Schedule fields (from sched):
 *   rounds = sum_t R_t;  moves_done, stuck_parts: sums;  max_batch: max;  node_rounds[q] = sum_t;
 *   node_last_round[q]   G_t + stage t's node_last_round[q] for the last stage t with a batch on q; 0 if none;
 *   part_done_round[p]   -1 if p is stuck in any stage; else G_t + stage t's part_done_round[p] for the last stage t
 *                        where p has ops; 0 if it never has ops.
 * Exposure fields (need expo; zero without it):
 *   peak[m] = max_t;  peak_stage[m], peak_round[m]: the first stage that reaches the peak and that stage's peak round;
 *   area[m] = sum_t - a map that ends stage t and begins stage t + 1 is counted in both;
 *   part_min_copies[p]   min over the stages whose begMap holds p; -1 if none;
 *   part_no_top[p] = sum_t;  part_flags[p]: OR over the stages;
 *   dom_peak[v] = max_t;  dom_peak_stage[v], dom_peak_round[v]: the first stage that reaches it and that stage's round.
 *
 * No value depends on n, max_concurrent, the wave size, the engine, the number of devices or the other move_conc.
 *
 * Errors, all before any device work, naming "chain i, stage t" or the index k: everything blance_plan_chains and
 * blance_plan_scenarios_exposure reject (with audit and expo optional as there: audit NULL = no audit, expo NULL = no
 * exposure); net_sched or net_expo without net, net_expo or a span exposure array without expo
 * (BLANCE_ERR_INVALID_ARG); a dom_peak / dom_peak_round of expo, net_expo or span with 2 x 17 x 2 x n_slots x n_parts
 * >= 2^31 (BLANCE_ERR_UNSUPPORTED; every stage shares the layout, so the bound is the same for each).  A NULL ctx
 * checks everything and then returns BLANCE_ERR_INVALID_ARG.  The span accumulators are priced into the wave size
 * next to the audit, exposure and net buffers (DESIGN.md section 15). */
typedef struct blance_chain_span_out {
  int64_t  rounds, moves_done, stuck_parts;
  int32_t  max_batch;
  int32_t* node_rounds;              /* [n_node_ids] */
  int64_t* node_last_round;          /* [n_node_ids] */
  int64_t* part_done_round;          /* [n_parts] */
  int64_t  peak[BLANCE_EXPO_N];
  int32_t  peak_stage[BLANCE_EXPO_N];
  int32_t  peak_round[BLANCE_EXPO_N];
  int64_t  area[BLANCE_EXPO_N];
  int32_t* part_min_copies;          /* [n_parts] */
  int32_t* part_no_top;              /* [n_parts] */
  uint8_t* part_flags;               /* [n_parts] */
  int64_t* dom_peak;                 /* [V] */
  int32_t* dom_peak_stage;           /* [V] */
  int32_t* dom_peak_round;           /* [V] */
} blance_chain_span_out;

int blance_plan_chains_exposure(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages,
                                const blance_chain_stage* stages /* [n][n_stages] */, const blance_scenario_opts* opts /* [n] or NULL */,
                                int32_t favor_min_nodes, int32_t max_concurrent,
                                int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                                blance_scenario_out* out /* [n][n_stages] */, blance_chain_out* net /* [n] or NULL */,
                                blance_scenario_schedule_out* sched /* [n][n_stages][n_move_conc] */,
                                const blance_audit_opts* aopts, blance_audit_out* audit /* [n][n_stages] or NULL */,
                                const blance_audit_opts* eopts /* forest only, flags must be 0; NULL = nodes only */,
                                int32_t series_cap, blance_exposure_out* expo /* [n][n_stages][n_move_conc] or NULL */,
                                blance_scenario_schedule_out* net_sched /* [n][n_move_conc] or NULL, needs net */,
                                blance_exposure_out* net_expo /* [n][n_move_conc] or NULL, needs net and expo */,
                                blance_chain_span_out* span /* [n][n_move_conc] or NULL */);

/* ---- plan options per chain stage (blance_plan_chains_ex) ---------------------------------------------------
 * blance_plan_chains_exposure where every STAGE has its own plan options: "add two nodes, then raise the replica
 * count", "bring in the new rack, then switch on the different-rack rule", "lose a node while the partition weights
 * change".  T = n_stages.  Stage t of chain i is
 *
 *     PlanNextMapEx(prev, assign, nodesAll_t, nodesToRemove_t, nodesToAdd_t, model, options_i_t)
 *
 * in the Go loop of blance_plan_chains, where options_i_t is the BASE's options with the groups of
 * stage_opts[i * T + t] substituted (as blance_plan_scenarios_ex does for one scenario) and stage t's NodeWeights.
 * The options are absolute, not cumulative: a group whose bit is clear at stage t is the base's, whatever an earlier
 * stage set; the partition weights of stage t are the base's with stage t's overrides applied.  From stage 2 on
 * extra_tot_first = extra_tot_rest as in blance_plan_chains, with the stage's own extra_tot_rest when its weight group
 * gives one.  stage_opts NULL: no options vary.  Every group keeps the rules of blance_plan_scenarios_ex (a
 * constraint within the base's slot range of its state, distinct override indices, weights <= 999999999, the count
 * bound), checked per stage.
 *
 * Per stage, the audit uses stage t's constraints and hierarchy rules and the exposure stage t's constraints.  The
 * net schedule and exposure (base prevMap -> the last stage's final map) use the LAST stage's constraints.  The span
 * folds the per-stage results as in blance_plan_chains_exposure.
 *
 * Arguments and outputs are those of blance_plan_chains_exposure, with opts [n] replaced by stage_opts [n][n_stages].
 * With stage_opts[i * T + t] = opts[i] for every t the outputs equal blance_plan_chains_exposure's byte for byte.  The
 * schedule may be left out: n_move_conc = 0 with move_conc and sched NULL plans (and audits, with audit) without one,
 * and then expo, net_sched, net_expo and span must be NULL.
 *
 * Errors, all before any device work: everything blance_plan_chains_exposure rejects, an option group's error
 * naming "chain i, stage t" (the audit model check too); expo, net_sched, net_expo or span without a schedule
 * (BLANCE_ERR_INVALID_ARG).  A member of a wave is laid out and priced by the largest of its stages (hierarchy masks,
 * rules and weight changes), so the automatic wave size holds at every stage (DESIGN.md section 16). */
int blance_plan_chains_ex(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages,
                          const blance_chain_stage* stages /* [n][n_stages] */,
                          const blance_scenario_opts* stage_opts /* [n][n_stages] or NULL */, int32_t favor_min_nodes,
                          int32_t max_concurrent, int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                          blance_scenario_out* out /* [n][n_stages] */, blance_chain_out* net /* [n] or NULL */,
                          blance_scenario_schedule_out* sched /* [n][n_stages][n_move_conc], or NULL without a schedule */,
                          const blance_audit_opts* aopts, blance_audit_out* audit /* [n][n_stages] or NULL */,
                          const blance_audit_opts* eopts, int32_t series_cap, blance_exposure_out* expo /* [n][n_stages][n_move_conc] or NULL */,
                          blance_scenario_schedule_out* net_sched /* [n][n_move_conc] or NULL, needs net */,
                          blance_exposure_out* net_expo /* [n][n_move_conc] or NULL, needs net and expo */,
                          blance_chain_span_out* span /* [n][n_move_conc] or NULL */);

/* ---- what-if branches off the stages of a chain (blance_plan_chain_branches) ---------------------------------
 * "What if node X fails after stage 2 of the rolling upgrade?" for every candidate failure and every stage, in one
 * call: blance_plan_chains_ex for the trunk chains, plus branches that leave trunk chain `chain` after its stage
 * `after_stage` and plan n_branch_stages stages of their own on that stage's final map.
 *
 * Branch b's EQUIVALENT CHAIN is trunk chain br[b].chain's stages 0..after_stage with their stage_opts, followed by
 * the branch's stages and stage_opts.  br_out[b * n_branch_stages + u] and the matching br_sched / br_audit / br_expo
 * entries equal stage after_stage + 1 + u of blance_plan_chains_ex on the equivalent chain, byte for byte; br_net,
 * br_net_sched and br_net_expo equal that call's net, net_sched and net_expo.  after_stage = -1 branches from the base
 * map (the branch is then a chain of its own).  Options are absolute, as in blance_plan_chains_ex: a branch stage with
 * NULL options plans with the base's options, not the trunk stage's.  The trunk outputs equal blance_plan_chains_ex
 * with the same trunk arguments byte for byte, and n_branches = 0 is that call.  One node_has_mover, move_conc,
 * aopts, eopts and series_cap serve trunk and branches.  Nothing depends on n, max_concurrent, the wave size, the
 * engine or the number of devices.
 *
 * The trunk prefix is planned once: after stage t of a trunk wave, the branches that leave its members there are
 * forked from the wave's working map on the device (DESIGN.md section 17).  For T trunk stages and N one-stage branches
 * after every stage that is T + N.T stage plans, against N.T(T+3)/2 when each equivalent chain is its own call.
 *
 * Errors, all before any device work: everything blance_plan_chains_ex rejects, with the checks of its stages run on
 * each equivalent chain's branch stages and named "branch b, stage u"; n_branches < 0; n_branches > 0 with
 * n_branch_stages < 1 or a NULL br, br_out or stages; chain outside [0, n) or after_stage outside [-1, n_stages);
 * br_sched NULL with a schedule or given without one; br_expo without a schedule or without expo; br_net_expo without
 * br_expo; br_net_sched or br_net_expo without br_net (BLANCE_ERR_INVALID_ARG).  With ctx NULL the call returns the
 * first error, or BLANCE_ERR_INVALID_ARG for the NULL ctx.
 *
 * Not provided: spans for branches (the trunk's span is unchanged), branches of branches, and a mover set or
 * favor_min_nodes of a branch's own. */
typedef struct blance_chain_branch {
  int32_t chain;                           /* the trunk chain it leaves, in [0, n) */
  int32_t after_stage;                     /* -1: from the base map; t in [0, n_stages): from trunk stage t's final map */
  const blance_chain_stage* stages;        /* [n_branch_stages] */
  const blance_scenario_opts* stage_opts;  /* [n_branch_stages] or NULL (no option group set) */
} blance_chain_branch;

int blance_plan_chain_branches(blance_ctx* ctx, const blance_plan_in* base, int32_t n, int32_t n_stages,
                               const blance_chain_stage* stages /* [n][n_stages] */,
                               const blance_scenario_opts* stage_opts /* [n][n_stages] or NULL */, int32_t favor_min_nodes,
                               int32_t max_concurrent, int32_t n_move_conc, const int32_t* move_conc, const uint8_t* node_has_mover,
                               blance_scenario_out* out /* [n][n_stages] */, blance_chain_out* net /* [n] or NULL */,
                               blance_scenario_schedule_out* sched /* [n][n_stages][n_move_conc], or NULL without a schedule */,
                               const blance_audit_opts* aopts, blance_audit_out* audit /* [n][n_stages] or NULL */,
                               const blance_audit_opts* eopts, int32_t series_cap, blance_exposure_out* expo /* [n][n_stages][n_move_conc] or NULL */,
                               blance_scenario_schedule_out* net_sched /* [n][n_move_conc] or NULL, needs net */,
                               blance_exposure_out* net_expo /* [n][n_move_conc] or NULL, needs net and expo */,
                               blance_chain_span_out* span /* [n][n_move_conc] or NULL */,
                               int32_t n_branches, int32_t n_branch_stages, const blance_chain_branch* br /* [n_branches] */,
                               blance_scenario_out* br_out /* [n_branches][n_branch_stages] */,
                               blance_chain_out* br_net /* [n_branches] or NULL */,
                               blance_scenario_schedule_out* br_sched /* [n_branches][n_branch_stages][n_move_conc], or NULL without a schedule */,
                               blance_audit_out* br_audit /* [n_branches][n_branch_stages] or NULL */,
                               blance_exposure_out* br_expo /* [n_branches][n_branch_stages][n_move_conc] or NULL, needs expo */,
                               blance_scenario_schedule_out* br_net_sched /* [n_branches][n_move_conc] or NULL, needs br_net */,
                               blance_exposure_out* br_net_expo /* [n_branches][n_move_conc] or NULL, needs br_net and br_expo */);

void blance_moves_free(blance_ctx* ctx, blance_moves* moves);

#ifdef __cplusplus
}
#endif
#endif /* BLANCE_B200_H_ */
