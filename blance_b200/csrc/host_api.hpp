// blance_b200/csrc/host_api.hpp — host-side mirror of blance's public planner API.
//
// The reference is Go and no Go toolchain exists in this image, so the host side
// above the C ABI (include/blance_b200.h) is written in C++ and mirrors api.go
// name for name:
//
//   PartitionMap / Partition            api.go:24-36
//   PartitionModel / ...State           api.go:41-62
//   HierarchyRules / HierarchyRule      api.go:75-105
//   PlanNextMapOptions                  api.go:183-190
//   PlanNextMap / PlanNextMapEx         api.go:109-157   (body -> blance_plan_next_map)
//   NodeStateOp / CalcPartitionMoves    moves.go:17-46   (body -> blance_calc_partition_moves)
//
// It does what the cgo shim of INTEGRATION.md does in Go: intern strings into the
// flat int32 tables of the C ABI, call the CUDA library, rebuild the maps, format
// the warning strings (plan.go:232-234) and replay the caller-map mutation of
// plan.go:49-52.  There is no CPU fallback: the calls throw BlanceError when the
// CUDA library reports a failure (e.g. no device).
#pragma once

#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "blance_b200.h"

namespace blance {

using Strs = std::vector<std::string>;
using OptStrs = std::optional<Strs>;   // Go's nil slice = nullopt (plan.go:554, reflect.DeepEqual)
using NodesByState = std::unordered_map<std::string, OptStrs>;

struct Partition {                     // api.go:28-36
  std::string Name;
  ::blance::NodesByState NodesByState;
};
using PartitionMap = std::unordered_map<std::string, Partition>;   // api.go:24 (values, not pointers)

// The JSON wire form of a PartitionMap, byte for byte what Go's encoding/json produces for
// map[string]*Partition with the tags of api.go:30,35 (`json:"name"`, `json:"nodesByState"`): object keys sorted
// by their bytes, a nil slice as null, strings escaped with encoding/json's default (HTML-safe) rules.
// The per-partition objects are rendered in parallel for large maps.
std::string PartitionMapToJSON(const PartitionMap& m);
// The same for the flat result of a plan (rows -> JSON without building the PartitionMap first).
struct InternedPlan;
struct PlanOutBuffers;
std::string PlanResultToJSON(const InternedPlan& ip, const PlanOutBuffers& ob);

struct PartitionModelState { int Priority = 0; int Constraints = 0; };   // api.go:46-62
using PartitionModel = std::unordered_map<std::string, PartitionModelState>;

struct HierarchyRule { int IncludeLevel = 0; int ExcludeLevel = 0; };     // api.go:95-105
using HierarchyRules = std::unordered_map<std::string, std::vector<HierarchyRule>>;

struct PlanNextMapOptions {            // api.go:183-190
  std::optional<std::unordered_map<std::string, int>> ModelStateConstraints;
  std::optional<std::unordered_map<std::string, int>> PartitionWeights;
  std::optional<std::unordered_map<std::string, int>> StateStickiness;
  std::optional<std::unordered_map<std::string, int>> NodeWeights;
  std::optional<std::unordered_map<std::string, std::string>> NodeHierarchy;
  std::optional<::blance::HierarchyRules> HierarchyRules;
  // The package-level knobs of plan.go, which a C ABI cannot read from Go globals:
  int MaxIterationsPerPlan = 10;       // plan.go:21
  int NodeScoreBooster = BLANCE_BOOSTER_NONE;   // plan.go:693; enum blance_booster
  int Engine = BLANCE_ENGINE_AUTO;     // enum blance_engine (not in the reference; results do not depend on it)
};

using Warnings = std::unordered_map<std::string, Strs>;

struct BlanceError : std::runtime_error {
  int status;
  BlanceError(int st, const std::string& what) : std::runtime_error(what), status(st) {}
};

struct PlanStats {                     // not in the reference; what the GPU did
  int iters_run = 0;
  int converged = 0;
  int64_t steps = 0;
  float device_ms = 0, kernel_ms = 0, pass_ms = 0;
  // host wall time of the stages of PlanNextMapEx: maps -> tables, the C ABI call, tables -> map, plan.go:49-52
  double intern_ms = 0, call_ms = 0, unintern_ms = 0, mutate_ms = 0;
};

// api.go:147-157.  prevMap and partitionsToAssign are mutated as plan.go:49-52
// mutates them (they may be the same object).
PartitionMap PlanNextMapEx(PartitionMap& prevMap, PartitionMap& partitionsToAssign, const Strs& nodesAll,
                           const OptStrs& nodesToRemove, const OptStrs& nodesToAdd,
                           const PartitionModel& model, const PlanNextMapOptions& options,
                           Warnings* warnings, PlanStats* stats = nullptr);

// ---- what-if scenarios of one cluster (blance_plan_scenarios) ----------------------------------------------------
template <class T>
using ScenarioOpt = std::optional<std::optional<T>>;   // outer nullopt: the options' value; inner nullopt: nil

struct Scenario {
  OptStrs NodesToRemove;               // nullopt = nil
  OptStrs NodesToAdd;                  // nullopt = nil (plan.go:554)
  ScenarioOpt<std::unordered_map<std::string, int>> NodeWeights;
  ScenarioOpt<std::unordered_map<std::string, int>> ModelStateConstraints;
  ScenarioOpt<std::unordered_map<std::string, int>> StateStickiness;
  ScenarioOpt<std::unordered_map<std::string, int>> PartitionWeights;   // names outside the maps are ignored
  ScenarioOpt<std::unordered_map<std::string, std::string>> NodeHierarchy;
  ScenarioOpt<::blance::HierarchyRules> HierarchyRules;
};

// The rebalance schedule of one scenario at one MaxConcurrentPartitionMovesPerNode (blance_plan_scenarios_schedule):
// the lock-step model of blance_moves_schedule over the moves NodeOps counts; per node (by name, nonzero entries
// only) the rounds with a batch and 1 + the last such round.
struct ScenarioSchedule {
  int MaxConcurrentPartitionMovesPerNode = 0;
  int Rounds = 0, MaxBatch = 0;
  int64_t MovesDone = 0, StuckParts = 0;
  std::unordered_map<std::string, int> NodeRounds, NodeLastRound;
};

// The audit of one map (include/blance_b200.h, "auditing a partition map"), by name; zero counts are left out.
struct MapAudit {
  std::unordered_map<std::string, int64_t> ShortSlots, OverSlots;                 // per model state
  std::unordered_map<std::string, std::vector<int64_t>> RuleMiss, RuleTested;     // per state with rules: one entry per rule, in rule order
  std::unordered_map<std::string, int64_t> DomTop, DomAll, DomCopies;             // per node or NodeHierarchy name
  int64_t ShortParts = 0, RuleMissParts = 0, NoTopParts = 0;
  bool HasFailoverSpread = false;      // the three fields below were asked for
  std::unordered_map<std::string, std::unordered_map<std::string, int32_t>> FailoverSpread;   // n2n[a][b] by name
  int32_t FailoverMax = 0;             // the largest entry, and the lowest (a, b) in node-id order that holds it
  std::string FailoverMaxFrom, FailoverMaxTo;
  std::unordered_map<std::string, int> PartFlags;                                 // bit 0 short, 1 rule miss, 2 no top node
};

// AuditMap audits `map` against `model` as PlanNextMapEx would read it with `options`: ModelStateConstraints
// override the constraints, HierarchyRules over NodeHierarchy are the rules checked (none when HierarchyRules is
// nil), and NodeHierarchy is also the fault-domain forest: the node names first, then every other name it mentions;
// a node absent from it, or whose parent is "", is its own root (nil: every node is its own domain).  nodesAll says
// which names are nodes the planner may pick (a node outside it never complies with a rule).  failoverSpread asks
// for the failover matrix.  Throws BlanceError for what blance_map_audit rejects (a cycle in NodeHierarchy, a name
// more than 16 levels below its root) and without a device.
MapAudit AuditMap(const PartitionMap& map, const Strs& nodesAll, const PartitionModel& model,
                  const PlanNextMapOptions& options, bool failoverSpread);

struct ScenarioResult {
  int iters_run = 0, converged = 0;
  int64_t steps = 0, sticky_steps = 0, parts_moved = 0, ops_total = 0, warn_parts = 0;
  // CalcPartitionMoves(prevMap row -> next row) of every assigned partition, counted per node and op name
  // ("add", "del", "promote", "demote"); nonzero counts only
  std::unordered_map<std::string, std::unordered_map<std::string, int64_t>> NodeOps;
  // countStateNodes (plan.go:374-399) of the final map per model state and node; nonzero loads only
  std::unordered_map<std::string, std::unordered_map<std::string, int64_t>> StateNodeLoad;
  bool HasMap = false;                 // the scenario was listed in wantMaps
  PartitionMap NextMap;                // as PlanNextMapEx returns it
  Warnings NextWarnings;
  std::vector<ScenarioSchedule> Schedules;   // one per scheduleConcurrency value; empty without them
  std::optional<MapAudit> Audit;       // with `audit`: the audit of the scenario's final map
};

// PlanNextMapScenarios' audit request: every result's Audit is AuditMap of that scenario's final map (prevMap with
// every assigned partition replaced by its next row) under the scenario's own constraints and hierarchy rules
// (blance_plan_scenarios_audit).  The fault-domain forest is the options' NodeHierarchy for every scenario.
struct ScenarioAudit { bool FailoverSpread = false; };

// Scenario i is PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, NodesToRemove_i, NodesToAdd_i, model, options
// with the scenario's NodeWeights, ModelStateConstraints, StateStickiness, PartitionWeights, NodeHierarchy and
// HierarchyRules substituted where it sets them).  Unlike PlanNextMapEx (plan.go:49-52), the caller's maps are NOT
// mutated: a what-if has no side effects.  The maps are interned once, each state's slot range as wide as the
// largest constraint of any scenario; a scenario's partition weights travel as the per-partition difference to the
// options' weights (blance_plan_scenarios_ex).  A scenario the reference would panic on (plan.go:544) or the device
// cannot plan (constraints above 16) throws BlanceError naming its index before any device work.  NextMap /
// NextWarnings are filled for the indices in wantMaps; maxConcurrent as in blance_plan_scenarios.
// scheduleConcurrency non-empty: each result's Schedules holds the rebalance schedule at each value
// (blance_plan_scenarios_schedule), with the nodesAll names as the movers, as OrchestrateSchedule has them.  One
// difference to OrchestrateSchedule: partitions are walked in interning order (the name rule of plan.go:519-528), where
// OrchestrateSchedule walks them in byte order of their names.  Both are valid instances of Go's map order, and they
// agree whenever the names sort the same under both rules.
std::vector<ScenarioResult> PlanNextMapScenarios(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                                 const Strs& nodesAll, const PartitionModel& model,
                                                 const PlanNextMapOptions& options, const std::vector<Scenario>& scenarios,
                                                 bool favorMinNodes, const std::vector<int>& wantMaps, int maxConcurrent,
                                                 const std::vector<int>& scheduleConcurrency = {},
                                                 const ScenarioAudit* audit = nullptr);

// ---- chains of cluster changes (blance_plan_chains) --------------------------------------------------------------
struct ChainStage {
  OptStrs NodesToRemove;               // nullopt = nil
  OptStrs NodesToAdd;                  // nullopt = nil (plan.go:554)
  ScenarioOpt<std::unordered_map<std::string, int>> NodeWeights;   // outer nullopt: the chain's / the options' value
  // This stage's nodesAll, a subset of the universe (PlanNextMapChains' nodesAll); it is always used in universe order.
  // nullopt: the previous stage's members minus its NodesToRemove, plus this stage's NodesToAdd that are in the
  // universe; the first stage's default is the whole universe.
  OptStrs NodesAll;
};

struct Chain {
  // The plan options of every stage of the chain: the option fields of a Scenario (ModelStateConstraints,
  // StateStickiness, PartitionWeights, NodeHierarchy, HierarchyRules, and NodeWeights unless a stage sets its own).
  // Its NodesToRemove / NodesToAdd are not read.
  Scenario Options;
  std::vector<ChainStage> Stages;
};

struct ChainResult {
  std::vector<ScenarioResult> Stages;  // one per stage, as PlanNextMapScenarios' results; "prev row" = that stage's prevMap
  // CalcPartitionMoves from the base prevMap row (empty when absent) to the last stage's next row, every assigned
  // partition: per node and op name (nonzero only), the total and the partitions with at least one op
  std::unordered_map<std::string, std::unordered_map<std::string, int64_t>> NetNodeOps;
  int64_t NetOpsTotal = 0, NetPartsMoved = 0;
};

// Chain i is the Go loop of include/blance_b200.h over its stages: stage t is PlanNextMapEx(prev, assign, nodesAll_t,
// NodesToRemove_t, NodesToAdd_t, model, options with chain i's option fields and stage t's NodeWeights), then prev =
// prev with every entry of next replaced and assign = next.  nodesAll is the UNIVERSE: every stage's nodesAll is a
// subset of it in its order, so a node that leaves and comes back keeps its position.  The caller's maps are NOT
// mutated; they are interned once.  Every chain has the same number of stages (>= 1).  A stage the reference would
// panic on (a removal in the first stage with assigned partitions absent from prevMap, plan.go:544), a NodesAll name
// outside the universe or chains of different lengths throw BlanceError naming the chain and stage before any device
// work.  Stage maps (NextMap / NextWarnings) are filled for the chains listed in wantMaps.
std::vector<ChainResult> PlanNextMapChains(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                           const Strs& nodesAll, const PartitionModel& model,
                                           const PlanNextMapOptions& options, const std::vector<Chain>& chains,
                                           bool favorMinNodes, const std::vector<int>& wantMaps, int maxConcurrent);

struct NodeStateOp { std::string Node, State, Op; };   // moves.go:17-21

// moves.go:41-46 for one partition (a batch of one on the device).
std::vector<NodeStateOp> CalcPartitionMoves(const Strs& states, const NodesByState& begNodesByState,
                                            const NodesByState& endNodesByState, bool favorMinNodes);

// The vectorised form: every partition of `beg` U `end` in one launch.
std::unordered_map<std::string, std::vector<NodeStateOp>> CalcPartitionMovesMap(
    const Strs& states, const PartitionMap& beg, const PartitionMap& end, bool favorMinNodes);

struct OrchestratorOptions {           // orchestrate.go:112-118
  int MaxConcurrentPartitionMovesPerNode = 0;
  bool FavorMinNodes = false;
};

struct AssignPartitionsCall {          // the arguments of one AssignPartitionsFunc call (orchestrate.go:96-100)
  std::string Node;
  Strs Partitions, States, Ops;
};

// The rebalance OrchestrateMoves(model, options, nodesAll, begMap, endMap, assign, LowestWeightPartitionMoveForNode)
// would run, under the lock-step model of blance_moves_schedule (include/blance_b200.h), computed on the device in
// one call: result[r] lists round r's AssignPartitionsFunc calls in node-id order (nodesAll first, then the other
// nodes in first-appearance order), each with its partitions, states and ops in pick order.  Partitions are
// begMap's keys indexed in byte order of their names; move lists are CalcPartitionMoves(sortStateNames(model), ...)
// as orchestrate.go:273-287 seeds them; a node outside nodesAll has no mover, so a partition whose next move is on
// it never advances.  len(begMap) != len(endMap) throws BlanceError with OrchestrateMoves' message.
std::vector<std::vector<AssignPartitionsCall>> OrchestrateSchedule(const PartitionModel& model, const OrchestratorOptions& options,
                                                                   const Strs& nodesAll, const PartitionMap& begMap,
                                                                   const PartitionMap& endMap);

// The exposure of that rebalance (blance_moves_exposure, include/blance_b200.h): the same move lists and schedule as
// OrchestrateSchedule, and the maps M_0 .. M_R it passes through counted per round.  Constraints are the model's
// Constraints (0 for state names outside the model), the top state is topPriorityStateName (plan.go:126-132; ties go
// to the first name in ascending order), and nodeHierarchy is the fault-domain forest as AuditMap builds it from
// NodeHierarchy (nil: every node is its own domain).  Metric-keyed fields ("NO_TOP", "MULTI_TOP", "SHORT",
// "ONE_COPY", "NO_COPY", "COPIES") hold every metric; vertex- and partition-keyed fields hold nonzero entries only
// (a partition absent from PartMinCopies had no copy at some round; DomPeakRound lists the vertices of DomPeak).
// Throws BlanceError for what OrchestrateSchedule or blance_moves_exposure rejects (e.g. more than 8 state names).
struct ExposureResult {
  int32_t Rounds = 0;
  std::unordered_map<std::string, std::vector<int64_t>> Series;   // [Rounds + 1] per metric
  std::unordered_map<std::string, int64_t> Peak, Area;
  std::unordered_map<std::string, int32_t> PeakRound;
  std::unordered_map<std::string, int64_t> DomPeak;               // per node or NodeHierarchy name
  std::unordered_map<std::string, int32_t> DomPeakRound;
  std::unordered_map<std::string, int32_t> PartMinCopies, PartNoTop, PartFlags;   // per partition; flags: bit m = metric m
  float KernelMs = 0.f;
};

ExposureResult OrchestrateExposure(const PartitionModel& model, const OrchestratorOptions& options, const Strs& nodesAll,
                                   const PartitionMap& begMap, const PartitionMap& endMap,
                                   const std::optional<std::unordered_map<std::string, std::string>>& nodeHierarchy);

// ---------------------------------------------------------------------------------
// The interning layer, exposed so that tests can drive the SAME tables through the
// CPU oracle and compare array for array.

struct InternedPlan {
  // name tables
  Strs node_names;        // [n_node_ids]
  Strs state_names;       // [n_states] in sortStateNames order
  Strs part_names;        // [n_parts] in the name-rule order of plan.go:519-528,512
  // tables (owning storage for the pointers in `in`)
  std::vector<int32_t> state_priority, state_constraints, state_slot_off, state_stickiness;
  std::vector<uint8_t> state_has_stickiness;
  std::vector<uint8_t> node_removed, node_added, node_has_weight;
  std::vector<int32_t> node_weight;
  std::vector<uint8_t> part_in_prev, part_in_assign, part_has_weight;
  std::vector<int32_t> part_weight, part_name_rank;
  std::vector<int32_t> prev_rows, cur_rows;
  std::vector<uint8_t> prev_shape, cur_shape;
  std::vector<int32_t> extra_tot_first, extra_tot_rest;
  std::vector<int32_t> extra_part, extra_node;   // the prevMap entries under non-model states behind extra_tot_*
  std::vector<int32_t> rule_off;
  std::vector<uint32_t> ie_mask;
  blance_plan_in in{};    // points into the vectors above
};

std::unique_ptr<InternedPlan> InternPlan(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                         const Strs& nodesAll, const OptStrs& nodesToRemove,
                                         const OptStrs& nodesToAdd, const PartitionModel& model,
                                         const PlanNextMapOptions& options);

struct PlanOutBuffers {
  std::vector<int32_t> next_rows;
  std::vector<uint8_t> next_shape, warn;
  blance_plan_out out{};
  explicit PlanOutBuffers(const InternedPlan& ip);
};

// rows -> PartitionMap of the assigned partitions, plus the warning strings.
PartitionMap UninternPlan(const InternedPlan& ip, const PlanOutBuffers& ob, Warnings* warnings);

// The blance_plan_in of scenario `index` of PlanNextMapScenarios: the shared base tables with that scenario's node
// fields and plan options substituted, its weight overrides applied (so a CPU oracle can run on exactly the tables
// the device plans).
std::unique_ptr<InternedPlan> InternScenario(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                             const Strs& nodesAll, const PartitionModel& model,
                                             const PlanNextMapOptions& options, const std::vector<Scenario>& scenarios,
                                             size_t index);

// plan.go:49-52: store the partitions of `next` into the caller's maps (they may be the same object).
void ReplayCallerMutation(const PartitionMap& next, PartitionMap& prevMap, PartitionMap& partitionsToAssign);

// The marshalling layer (InternPlan, UninternPlan, ReplayCallerMutation) splits maps of 32 768 partitions
// or more over host threads: min(16, hardware threads) by default, BLANCE_HOST_THREADS in the environment,
// or this call (0 = back to the default).  Results do not depend on the thread count.
void SetHostThreads(int n);
int HostThreads();

// The fault-domain forest AuditMap passes as blance_audit_opts.domain_parent: vertex names (ip's node ids first, then
// every other name of nodeHierarchy in byte order) and each vertex's parent index, -1 for a root (a name without a
// parent, or whose parent is "").  nodeHierarchy nil: the node names and an empty parent array (nodes only).
void AuditForest(const InternedPlan& ip, const std::optional<std::unordered_map<std::string, std::string>>& nodeHierarchy,
                 Strs* names, std::vector<int32_t>* parent);

// The process-wide context the host API runs on (created on first use).
blance_ctx* DefaultContext();

}  // namespace blance
