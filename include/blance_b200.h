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
 * there is no collective in the data path); every other entry point runs on device_ids[0]. */
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
  const uint8_t* node_removed;          /* in nodesToRemove */
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
 * 2^30, partition weights within the "%10d" rule of plan.go:539, rule_off monotone.  The planning entry points do
 * NOT scan the contents (it would sit in the timed path of every call): a binding that does not trust its own
 * marshalling calls this first.  Returns BLANCE_OK / BLANCE_ERR_INVALID_ARG / BLANCE_ERR_UNSUPPORTED; msg (may be
 * NULL) receives the reason, truncated to msg_cap bytes. */
int blance_plan_in_check(const blance_plan_in* in, char* msg, int32_t msg_cap);

/* Host buffers in, host buffers out.  If prevMap and partitionsToAssign must be
 * mutated as plan.go:49-52 does, the caller copies next_rows back when
 * iters_run >= 2 || !converged. */
int blance_plan_next_map(blance_ctx* ctx, const blance_plan_in* in, blance_plan_out* out);

/* n independent instances (multi-tenant rebalance fan-out); instance i uses
 * in[i] / out[i].  All instances of a device run concurrently (one CTA each per pass); a multi-device
 * context spreads them over its GPUs. */
int blance_plan_next_map_batch(blance_ctx* ctx, int32_t n, const blance_plan_in* in, blance_plan_out* out);

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
 * partitions together (the size of the op_* arrays blance_moves_fetch fills). */
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
void blance_moves_free(blance_ctx* ctx, blance_moves* moves);

#ifdef __cplusplus
}
#endif
#endif /* BLANCE_B200_H_ */
