"""Python face of the host API.  Mirrors the reference's exported names:

    PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, options)
        -> (nextMap, warnings)                                    api.go:147-157
    PlanNextMap(..., modelStateConstraints, partitionWeights, stateStickiness, nodeWeights,
                nodeHierarchy, hierarchyRules) -> (nextMap, warnings)   api.go:109-132 (deprecated wrapper)
    CalcPartitionMoves(states, begNodesByState, endNodesByState, favorMinNodes) -> [NodeStateOp]   moves.go:41-46
    OrchestrateSchedule(model, options, nodesAll, begMap, endMap) -> rounds of AssignPartitionsFunc calls
        (the lock-step model of OrchestrateMoves, orchestrate.go:240-591; include/blance_b200.h)
    OrchestrateExposure(model, options, nodesAll, begMap, endMap, nodeHierarchy) -> the maps those rounds pass
        through, counted per round (blance_moves_exposure)
    OrchestrateLoad(model, options, nodesAll, begMap, endMap, partitionWeights) -> each node's load on those maps:
        start, end and peak (blance_moves_load)

A PartitionMap is {partitionName: {stateName: [nodeName, ...] | None}}; a
PartitionModel is {stateName: (priority, constraints)}; HierarchyRules is
{stateName: [(includeLevel, excludeLevel), ...]}.  prevMap and
partitionsToAssign are mutated in place exactly as plan.go:49-52 mutates them.
"""
import collections
import ctypes
import dataclasses
import typing

from . import _host
from . import build as _build

from .abi import BlanceError     # base class; _host.BlanceError derives from it
BOOSTER_NONE = 0
BOOSTER_CBGT_MAX = 1     # cbgt's max(float64(-w), stickiness), control_test.go:19-26

NodeStateOp = collections.namedtuple("NodeStateOp", ["Node", "State", "Op"])   # moves.go:17-21


@dataclasses.dataclass
class PlanNextMapOptions:          # api.go:183-190 (+ the package-level hooks of plan.go:21,693)
    ModelStateConstraints: typing.Optional[dict] = None
    PartitionWeights: typing.Optional[dict] = None
    StateStickiness: typing.Optional[dict] = None
    NodeWeights: typing.Optional[dict] = None
    NodeHierarchy: typing.Optional[dict] = None
    HierarchyRules: typing.Optional[dict] = None
    MaxIterationsPerPlan: int = 10
    NodeScoreBooster: int = BOOSTER_NONE
    Engine: int = 0


def _replace(dst, src):
    dst.clear()
    dst.update(src)


def PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, options=None,
                  stats=None):
    o = options or PlanNextMapOptions()
    same = prevMap is partitionsToAssign
    r = _host.PlanNextMapEx(prevMap, None if same else partitionsToAssign, list(nodesAll),
                            None if nodesToRemove is None else list(nodesToRemove),
                            None if nodesToAdd is None else list(nodesToAdd),
                            {k: tuple(v) for k, v in model.items()},
                            o.ModelStateConstraints, o.PartitionWeights, o.StateStickiness, o.NodeWeights,
                            o.NodeHierarchy,
                            None if o.HierarchyRules is None else {k: [tuple(x) for x in v] for k, v in o.HierarchyRules.items()},
                            o.NodeScoreBooster, o.MaxIterationsPerPlan, o.Engine)
    _replace(prevMap, r["prev_map"])                 # plan.go:49-52
    if not same:
        _replace(partitionsToAssign, r["partitions_to_assign"])
    if stats is not None:
        stats.update({k: r[k] for k in ("iterations", "converged", "steps", "device_ms", "kernel_ms", "pass_ms")})
    return r["next_map"], r["warnings"]


def PlanNextMap(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model,
                modelStateConstraints=None, partitionWeights=None, stateStickiness=None, nodeWeights=None,
                nodeHierarchy=None, hierarchyRules=None):
    return PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model,
                         PlanNextMapOptions(modelStateConstraints, partitionWeights, stateStickiness, nodeWeights,
                                            nodeHierarchy, hierarchyRules))


def _rules_arg(rules):
    return None if rules is None else {k: [tuple(x) for x in v] for k, v in rules.items()}


# the optional per-scenario option keys, in the order _host expects their (has_key, value) pairs
_SCENARIO_OPTION_KEYS = (("nodeWeights", dict), ("modelStateConstraints", dict), ("stateStickiness", dict),
                         ("partitionWeights", dict), ("nodeHierarchy", dict), ("hierarchyRules", _rules_arg))


def _scenario_tuples(scenarios):
    out = []
    for i, sc in enumerate(scenarios):
        missing = {"nodesToRemove", "nodesToAdd"} - set(sc)
        if missing:
            raise ValueError("scenario %d lacks %s" % (i, ", ".join(sorted(missing))))
        rm, ad = sc["nodesToRemove"], sc["nodesToAdd"]
        t = [None if rm is None else list(rm), None if ad is None else list(ad)]
        for key, conv in _SCENARIO_OPTION_KEYS:
            t += [key in sc, None if sc.get(key) is None else conv(sc[key])]
        out.append(tuple(t))
    return out


def _option_kwargs(o):
    return dict(model_state_constraints=o.ModelStateConstraints, partition_weights=o.PartitionWeights,
                state_stickiness=o.StateStickiness, node_weights=o.NodeWeights, node_hierarchy=o.NodeHierarchy,
                hierarchy_rules=None if o.HierarchyRules is None else {k: [tuple(x) for x in v] for k, v in o.HierarchyRules.items()},
                booster=o.NodeScoreBooster, max_iterations=o.MaxIterationsPerPlan, engine=o.Engine)


def PlanNextMapScenarios(prevMap, partitionsToAssign, nodesAll, model, options=None, scenarios=(), favorMinNodes=False,
                         wantMaps=(), maxConcurrent=0, scheduleConcurrency=(), audit=None, exposure=None):
    """What-if variants of one cluster, planned side by side on the device.  Scenario i is
    PlanNextMapEx(prevMap, partitionsToAssign, nodesAll, sc["nodesToRemove"], sc["nodesToAdd"], model, options with
    the scenario's plan options substituted): both node-set keys are required (None = nil).  The optional keys
    "nodeWeights", "modelStateConstraints", "stateStickiness", "partitionWeights", "nodeHierarchy" and
    "hierarchyRules" replace the options field of the same name; a missing key inherits it, None means nil.
    The caller's maps are NOT mutated.

    Returns one dict per scenario: iterations, converged, steps, sticky_steps, parts_moved, ops_total, warn_parts,
    node_ops {node: {op: count}} and state_node_load {state: {node: load}} (nonzero entries only), plus next_map and
    warnings for the indices in wantMaps.

    scheduleConcurrency (a list of MaxConcurrentPartitionMovesPerNode values) adds a "schedules" list to every dict:
    the lock-step rebalance schedule of OrchestrateSchedule over the moves node_ops counts, one dict per value with
    MaxConcurrentPartitionMovesPerNode, Rounds, MovesDone, StuckParts, MaxBatch, and NodeRounds / NodeLastRound
    {node: rounds with a batch / 1 + the last such round} (nonzero entries only).  The movers are the nodesAll names.
    Partitions are walked in interning order (the name rule of plan.go:519-528) where OrchestrateSchedule walks them in
    byte order: both are valid instances of Go's map order and agree whenever the names sort the same under both.

    audit (None = no audit, exactly the results above; or a dict with the optional key "failoverSpread") adds an
    "audit" dict to every result: AuditMap of that scenario's final map (prevMap with every assigned partition
    replaced by its next row) under the scenario's own constraints and hierarchy rules, computed inside the sweep
    without copying the map out.  The fault domains are the options' NodeHierarchy for every scenario.

    exposure (None = none; or a dict with the optional key "seriesCap", default 0) needs scheduleConcurrency and adds
    an "exposures" list to every result, one dict per value, shaped as OrchestrateExposure's: the exposure of that
    scenario's rebalance (begMap = prevMap plus an empty entry for every assigned partition it lacks, endMap = the
    final map) under the scenario's own constraints, with the options' NodeHierarchy as the fault domains.  "series"
    holds the first min(rounds + 1, seriesCap) values per metric; rounds, peak, peak_round and area are complete."""
    o = options or PlanNextMapOptions()
    same = prevMap is partitionsToAssign
    return _host.PlanNextMapScenarios(prevMap, None if same else partitionsToAssign, list(nodesAll),
                                      {k: tuple(v) for k, v in model.items()}, _scenario_tuples(scenarios),
                                      bool(favorMinNodes), [int(i) for i in wantMaps], int(maxConcurrent), **_option_kwargs(o),
                                      schedule_concurrency=[int(c) for c in scheduleConcurrency],
                                      audit=None if audit is None else bool(audit.get("failoverSpread", False)),
                                      exposure_series_cap=None if exposure is None else int(exposure.get("seriesCap", 0)))


def PlanNextMapChains(prevMap, partitionsToAssign, nodesAll, model, options=None, chains=(), favorMinNodes=False,
                      wantMaps=(), maxConcurrent=0, scheduleConcurrency=(), audit=None, exposure=None, branches=None):
    """Chains of cluster changes, each stage planned on the map the stage before produced (blance_plan_chains).  Chain
    i runs the Go loop `next = PlanNextMapEx(prev, assign, nodesAll_t, nodesToRemove_t, nodesToAdd_t, model, options_i_t);
    prev = prev with every entry of next replaced; assign = next` over its stages.  nodesAll is the universe: a stage's
    nodesAll is a subset of it, always in its order.  A chain is a dict with "stages" (a list) and the optional option
    keys of PlanNextMapScenarios' scenarios ("nodeWeights", "modelStateConstraints", "stateStickiness",
    "partitionWeights", "nodeHierarchy", "hierarchyRules": missing inherits the options, None means nil), shared by
    its stages.  A stage is a dict with "nodesToRemove" and "nodesToAdd" (required, None = nil), an optional
    "nodesAll" and the same optional option keys: a stage's own value replaces the chain's for that stage only (the
    next stage starts from the chain's again).  Without "nodesAll", the previous stage's members minus its
    nodesToRemove plus this stage's nodesToAdd (the first stage: the whole universe).  Every chain has the same number
    of stages.  The caller's maps are NOT mutated.

    Returns one dict per chain: "stages", one dict per stage with the keys of PlanNextMapScenarios' results (next_map
    and warnings for the chains in wantMaps), and "net": node_ops, ops_total and parts_moved of CalcPartitionMoves
    from the base prevMap to the last stage's map.

    scheduleConcurrency, audit and exposure (as PlanNextMapScenarios; the movers are the universe) add "schedules",
    "audit" and "exposures" to every stage's dict, with that stage's prevMap as begMap.  Then "net" also gets
    "schedules" (and with exposure "exposures") of the direct rebalance from prevMap to the last stage's map, and each
    chain dict a "span" list, one dict per value: the chain's stages folded on one global round axis (rounds,
    moves_done, stuck_parts, max_batch; node_rounds / node_last_round {node: ...}; part_done_round {partition: ...,
    -1 = stuck in some stage}; with exposure peak / peak_stage / peak_round / area {metric: ...}, part_min_copies /
    part_no_top / part_flags {partition: ...}, dom_peak / dom_peak_stage / dom_peak_round {name: ...}), nonzero
    entries only.

    branches (blance_plan_chain_branches): a list of dicts with "chain" (the index of the chain it leaves),
    "afterStage" (the stage after which it leaves, -1 for the base map), "stages" (stage dicts as above, the same number
    in every branch) and an optional "wantMaps" (bool).  A branch is planned as stages afterStage + 1, ... of its
    equivalent chain: the chain's options and stages 0..afterStage followed by the branch's stages (so a branch stage
    without "nodesAll" starts from trunk stage afterStage's members).  The return is then (chains, branches): one dict
    per branch shaped like a chain's, without "span"."""
    o = options or PlanNextMapOptions()
    same = prevMap is partitionsToAssign

    def stage_tuples(where, stages):
        out = []
        for t, st in enumerate(stages):
            missing = {"nodesToRemove", "nodesToAdd"} - set(st)
            if missing:
                raise ValueError("%s, stage %d lacks %s" % (where, t, ", ".join(sorted(missing))))
            na = st.get("nodesAll")
            out.append((_scenario_tuples([st])[0], None if na is None else list(na)))
        return out

    cs = []
    for i, c in enumerate(chains):
        opts = {k: v for k, v in c.items() if k != "stages"}
        opts.update(nodesToRemove=None, nodesToAdd=None)
        cs.append((_scenario_tuples([opts])[0], stage_tuples("chain %d" % i, c["stages"])))
    bs = None if branches is None else [
        (int(b["chain"]), int(b["afterStage"]), stage_tuples("branch %d" % x, b["stages"]), bool(b.get("wantMaps", False)))
        for x, b in enumerate(branches)]
    return _host.PlanNextMapChains(prevMap, None if same else partitionsToAssign, list(nodesAll),
                                   {k: tuple(v) for k, v in model.items()}, cs, bool(favorMinNodes),
                                   [int(i) for i in wantMaps], int(maxConcurrent), **_option_kwargs(o),
                                   schedule_concurrency=[int(c) for c in scheduleConcurrency],
                                   audit=None if audit is None else bool(audit.get("failoverSpread", False)),
                                   exposure_series_cap=None if exposure is None else int(exposure.get("seriesCap", 0)),
                                   branches=bs)


def AuditMap(partitionMap, nodesAll, model, options=None, failoverSpread=False):
    """What the planner never reports about a finished map (include/blance_b200.h, "auditing a partition map"),
    counted on the device.  options (PlanNextMapOptions): ModelStateConstraints override the model's constraints;
    HierarchyRules over NodeHierarchy are the rules checked; NodeHierarchy is also the fault-domain forest (a node
    absent from it is its own root).  Returns a dict, zero counts left out:
      short_slots / over_slots {state: slots}, short_parts;
      rule_miss / rule_tested {state: [count per rule of that state]}, rule_miss_parts: placements the planner made by
        its silent fallback (plan.go:214-220), e.g. a replica in its primary's rack;
      dom_copies / dom_top / dom_all {node or hierarchy name: copies under it / partitions whose top node is under it /
        partitions that live under it alone}, no_top_parts;
      part_flags {partition: bit 0 short | bit 1 rule miss | bit 2 no top node};
      with failoverSpread: failover_spread {a: {b: copies on b of partitions whose top node is a}} and failover_max
        (count, a, b), the node that takes the most promotions when a fails."""
    o = options or PlanNextMapOptions()
    return _host.AuditMap(partitionMap, list(nodesAll), {k: tuple(v) for k, v in model.items()},
                          model_state_constraints=o.ModelStateConstraints, node_hierarchy=o.NodeHierarchy,
                          hierarchy_rules=_rules_arg(o.HierarchyRules), failover_spread=bool(failoverSpread))


def intern_scenario(prevMap, partitionsToAssign, nodesAll, model, options, scenarios, index):
    """The blance_plan_in of scenario `index` of PlanNextMapScenarios as an interned plan (_host.InternedPlan), for
    running a CPU oracle on exactly the tables the device plans."""
    o = options or PlanNextMapOptions()
    same = prevMap is partitionsToAssign
    return _host.intern_scenario(prevMap, None if same else partitionsToAssign, list(nodesAll),
                                 {k: tuple(v) for k, v in model.items()}, _scenario_tuples(scenarios), int(index),
                                 **_option_kwargs(o))


def CalcPartitionMoves(states, begNodesByState, endNodesByState, favorMinNodes):
    return [NodeStateOp(*t) for t in _host.CalcPartitionMoves(list(states), begNodesByState, endNodesByState,
                                                              bool(favorMinNodes))]


def CalcPartitionMovesMap(states, begMap, endMap, favorMinNodes):
    """Vectorised CalcPartitionMoves over two PartitionMaps: {partitionName: [NodeStateOp]}."""
    r = _host.CalcPartitionMovesMap(list(states), begMap, endMap, bool(favorMinNodes))
    return {k: [NodeStateOp(*t) for t in v] for k, v in r.items()}


@dataclasses.dataclass
class OrchestratorOptions:         # orchestrate.go:112-118
    MaxConcurrentPartitionMovesPerNode: int = 0
    FavorMinNodes: bool = False


AssignPartitionsCall = collections.namedtuple("AssignPartitionsCall", ["Node", "Partitions", "States", "Ops"])


def OrchestrateSchedule(model, options, nodesAll, begMap, endMap):
    """The rebalance OrchestrateMoves(model, options, nodesAll, begMap, endMap, ..., LowestWeightPartitionMoveForNode)
    runs, under the lock-step model of blance_moves_schedule, computed on the device: one list per round of
    AssignPartitionsCall(Node, Partitions, States, Ops) in node-id order (nodesAll first), each in pick order.  A
    node outside nodesAll has no mover: a partition whose next move is on it never advances."""
    o = options or OrchestratorOptions()
    r = _host.OrchestrateSchedule({k: tuple(v) for k, v in model.items()}, int(o.MaxConcurrentPartitionMovesPerNode),
                                  bool(o.FavorMinNodes), list(nodesAll), begMap, endMap)
    return [[AssignPartitionsCall(*c) for c in rnd] for rnd in r]


def OrchestrateExposure(model, options, nodesAll, begMap, endMap, nodeHierarchy=None):
    """Is the data safe while the rebalance of OrchestrateSchedule(model, options, nodesAll, begMap, endMap) runs?  The
    maps M_0 .. M_R it passes through under the lock-step model (M_t: after t rounds of AssignPartitionsFunc calls),
    counted on the device (blance_moves_exposure, include/blance_b200.h).  Constraints are the model's, the top state
    is the model's lowest priority (ties: first name), nodeHierarchy ({child: parent}, as NodeHierarchy) the
    fault-domain forest (None: every node is its own domain).  Returns a dict:
      rounds R;  series {metric: [R + 1 values]}, peak / peak_round / area {metric: ...} for every metric of
        NO_TOP (no primary), MULTI_TOP (more primaries than the constraint), SHORT, ONE_COPY, NO_COPY, COPIES;
      dom_peak / dom_peak_round {node or hierarchy name: most partitions it alone held at one round / first such
        round}, part_min_copies / part_no_top / part_flags {partition: ...}: nonzero entries only;
      kernel_ms."""
    o = options or OrchestratorOptions()
    return _host.OrchestrateExposure({k: tuple(v) for k, v in model.items()}, int(o.MaxConcurrentPartitionMovesPerNode),
                                     bool(o.FavorMinNodes), list(nodesAll), begMap, endMap,
                                     None if nodeHierarchy is None else dict(nodeHierarchy))


def OrchestrateLoad(model, options, nodesAll, begMap, endMap, partitionWeights=None):
    """Does a node run out of room while the rebalance of OrchestrateSchedule(model, options, nodesAll, begMap, endMap)
    runs?  Each node's load on the maps M_0 .. M_R it passes through under the lock-step model, counted on the device
    (blance_moves_load, include/blance_b200.h).  A partition weighs partitionWeights[name] ({partition: weight}, as
    PartitionWeights), 1 when it has none.  Returns a dict:
      rounds R;  states {state: {node: {beg, end, peak, peak_round}}} and nodes {node: {...}} over all states (nonzero
        entries only): the load on M_0, on M_R, its largest value and the first round at it;
      over_max / over_node: the largest peak over both ends of one node (all states) and that node ("" without nodes);
      kernel_ms."""
    o = options or OrchestratorOptions()
    return _host.OrchestrateLoad({k: tuple(v) for k, v in model.items()}, int(o.MaxConcurrentPartitionMovesPerNode),
                                 bool(o.FavorMinNodes), list(nodesAll), begMap, endMap,
                                 None if partitionWeights is None else {k: int(v) for k, v in partitionWeights.items()})


# ---- the raw C ABI (ctypes) lives in abi.py; re-exported here for callers of the Python face -----------
from .abi import AUDIT_N2N, AuditOpts, AuditOut, EXPORTS, PlanIn, PlanOut, Scenario, ScenarioOpts, ScenarioOut, ScenarioScheduleOut, ScheduleOut, _I32_FIELDS, _PTR_FIELDS, capi  # noqa: E402,F401
