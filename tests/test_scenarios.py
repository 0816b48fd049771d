"""What-if scenarios of one cluster (PlanNextMapScenarios / blance_plan_scenarios), CPU side: the host layer's
per-scenario tables against the literal oracle, the semantics of the summaries, input checks and the ABI.  No
device needed (the device path is tests/test_scenarios_gpu.py)."""
import copy
import ctypes
import os
import subprocess
import tempfile

import pytest

import golden_util as G
from oracle_loader import fast_lib_path, literal
from randgen import random_instance

import blance_b200
from blance_b200 import _host, api

L = literal()
FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUTSIDE = "zz-not-in-nodesAll"


def options_of(kw):
    return blance_b200.PlanNextMapOptions(
        ModelStateConstraints=kw.get("model_state_constraints"), PartitionWeights=kw.get("partition_weights"),
        StateStickiness=kw.get("state_stickiness"), NodeWeights=kw.get("node_weights"),
        NodeHierarchy=kw.get("node_hierarchy"), HierarchyRules=kw.get("hierarchy_rules"),
        NodeScoreBooster=kw.get("booster", 0))


def scenario_kwargs(kw, sc):
    """The PlanNextMapEx arguments of scenario `sc` (deep copies: the reference mutates its maps)."""
    k = copy.deepcopy(kw)
    k["nodes_to_remove"] = copy.deepcopy(sc["nodesToRemove"])
    k["nodes_to_add"] = copy.deepcopy(sc["nodesToAdd"])
    if "nodeWeights" in sc:
        k["node_weights"] = copy.deepcopy(sc["nodeWeights"])
    return k


def removal_allowed(kw):
    """plan.go:544: a non-empty nodesToRemove needs every assigned partition in prevMap."""
    assign = kw["partitions_to_assign"]
    return assign is None or all(p in kw["prev_map"] for p in assign)


def make_scenarios(kw, seed):
    """3-6 variants: the case's own node sets, a single-node removal, a removed name outside nodesAll, nodesToAdd
    nil vs [], NodeWeights inherited / replaced / nil."""
    nodes = kw["nodes_all"]
    rm_ok = removal_allowed(kw)
    scs = [{"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": kw["nodes_to_add"]}]
    if rm_ok and nodes:
        scs.append({"nodesToRemove": [nodes[seed % len(nodes)]], "nodesToAdd": kw["nodes_to_add"]})
    if rm_ok:
        scs.append({"nodesToRemove": [OUTSIDE], "nodesToAdd": []})
    scs.append({"nodesToRemove": None, "nodesToAdd": None})
    scs.append({"nodesToRemove": [], "nodesToAdd": [], "nodeWeights": {n: (i % 4) - 1 for i, n in enumerate(nodes)}})
    scs.append({"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": nodes[:1], "nodeWeights": None})
    return scs[:3 + seed % 4] if len(scs) > 3 + seed % 4 else scs


def state_order(model):
    return L.state_name_sort(model, sorted(model))


def summary_reference(kw, next_map, warnings, favor_min_nodes=False):
    """The summaries of one scenario from the literal oracle's next map and the literal CalcPartitionMoves: per
    assigned partition CalcPartitionMoves(all model states, prevMap row over the model states (empty when absent),
    next row); countStateNodes over the model states of prevMap with the assigned rows replaced.  Zero entries are
    left out, as PlanNextMapScenarios leaves them out."""
    model = kw["model"]
    states = state_order(model)
    prev = kw["prev_map"]
    assign = kw["partitions_to_assign"] if kw["partitions_to_assign"] is not None else prev
    node_ops, parts_moved, ops_total = {}, 0, 0
    for p in assign:
        beg = {s: v for s, v in prev.get(p, {}).items() if s in model}
        ops = L.calc_partition_moves(states, beg, next_map.get(p, {}), favor_min_nodes)
        parts_moved += bool(ops)
        ops_total += len(ops)
        for node, _state, op in ops:
            node_ops.setdefault(node, {}).setdefault(op, 0)
            node_ops[node][op] += 1
    final = dict(prev)
    final.update(next_map)
    pw = kw.get("partition_weights")
    load = {}
    for p, nbs in final.items():
        w = pw.get(p, 1) if pw is not None else 1
        for s, nodes in nbs.items():
            if s not in model:
                continue
            for n in nodes or []:
                load.setdefault(s, {}).setdefault(n, 0)
                load[s][n] += w
    load = {s: {n: v for n, v in m.items() if v} for s, m in load.items()}
    load = {s: m for s, m in load.items() if m}
    return dict(node_ops=node_ops, parts_moved=parts_moved, ops_total=ops_total, state_node_load=load,
                warn_parts=len(warnings))


def check_scenarios(kw, scs):
    o = options_of(kw)
    prev, assign = kw["prev_map"], kw["partitions_to_assign"]
    for i, sc in enumerate(scs):
        ip = api.intern_scenario(prev, prev if assign is None else assign, kw["nodes_all"], kw["model"], o, scs, i)
        out = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, out.out_ptr) == 0
        next_map, warnings = _host.unintern_plan(ip, out)
        lit = L.plan_next_map_ex(**scenario_kwargs(kw, sc))
        if out.iters_run <= 0:
            next_map, warnings = {}, {}
        assert next_map == lit["next_map"], i
        assert warnings == lit["warnings"], i
        assert out.iters_run == lit["iterations"], i


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_scenario_tables_match_literal_oracle_golden(c):
    kw = G.plan_kwargs(c)
    check_scenarios(kw, make_scenarios(kw, c["index"]))


@pytest.mark.parametrize("chunk", range(6))
def test_scenario_tables_match_literal_oracle_random(chunk):
    for seed in range(chunk * 50, (chunk + 1) * 50):
        kw = random_instance(seed)
        check_scenarios(kw, make_scenarios(kw, seed))


def test_interning_is_independent_of_the_other_scenarios():
    """The node-id space holds every scenario's names, but a scenario's tables plan the same map either way."""
    kw = G.plan_kwargs(G.plan_cases()[0])
    scs = make_scenarios(kw, 1)
    o = options_of(kw)
    alone = api.intern_scenario(kw["prev_map"], kw["prev_map"] if kw["partitions_to_assign"] is None else kw["partitions_to_assign"],
                                kw["nodes_all"], kw["model"], o, scs[:1], 0)
    together = api.intern_scenario(kw["prev_map"], kw["prev_map"] if kw["partitions_to_assign"] is None else kw["partitions_to_assign"],
                                   kw["nodes_all"], kw["model"], o, scs, 0)
    maps = []
    for ip in (alone, together):
        out = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, out.out_ptr) == 0
        maps.append(_host.unintern_plan(ip, out))
    assert maps[0] == maps[1]
    assert together.n_node_ids >= alone.n_node_ids


# ---- summary semantics ----------------------------------------------------------------------------------------

def test_summary_reference_hand_counted():
    model = {"primary": (0, 1), "replica": (1, 1)}
    prev = {"0": {"primary": ["a"], "replica": ["b"]}, "1": {"primary": ["b"], "replica": ["c"]},
            "2": {"primary": ["c"], "dead": ["a"]}}
    assign = {"0": prev["0"], "1": prev["1"], "3": {}}
    nxt = {"0": {"primary": ["b"], "replica": ["c"]}, "1": {"primary": ["b"], "replica": ["c"]},
           "3": {"primary": ["a"], "replica": []}}
    kw = dict(prev_map=prev, partitions_to_assign=assign, model=model, partition_weights={"2": 5})
    r = summary_reference(kw, nxt, {"3": ["w"]})
    # "0": promote b (was a replica), del a, add c to replica; "1": nothing; "3" (not in prevMap): add a
    assert r["node_ops"] == {"b": {"promote": 1}, "a": {"del": 1, "add": 1}, "c": {"add": 1}}
    assert (r["parts_moved"], r["ops_total"], r["warn_parts"]) == (2, 4, 1)
    # final map: 0 p[b] r[c]; 1 p[b] r[c]; 2 p[c] (weight 5; "dead" is not a model state); 3 p[a]
    assert r["state_node_load"] == {"primary": {"b": 2, "c": 5, "a": 1}, "replica": {"c": 2}}


def test_summary_reference_on_golden_cases_is_consistent():
    for c in G.plan_cases():
        kw = G.plan_kwargs(c)
        lit = L.plan_next_map_ex(**copy.deepcopy(kw))
        r = summary_reference(kw, lit["next_map"], lit["warnings"])
        assert r["ops_total"] == sum(sum(v.values()) for v in r["node_ops"].values()), G.case_id(c)
        assert r["parts_moved"] <= len(lit["next_map"]), G.case_id(c)
        assert (r["parts_moved"] == 0) == (r["ops_total"] == 0), G.case_id(c)
        assert r["warn_parts"] == len(lit["warnings"]), G.case_id(c)


# ---- invalid input ----------------------------------------------------------------------------------------------

def test_a_scenario_the_reference_panics_on_is_rejected_by_index():
    prev = {"0": {"primary": ["a"]}}
    assign = {"0": {"primary": ["a"]}, "1": {}}          # "1" is missing from prevMap
    scs = [{"nodesToRemove": [], "nodesToAdd": None}, {"nodesToRemove": ["a"], "nodesToAdd": None}]
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: "):
        blance_b200.PlanNextMapScenarios(prev, assign, ["a", "b"], {"primary": (0, 1)}, None, scs)
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: "):
        api.intern_scenario(prev, assign, ["a", "b"], {"primary": (0, 1)}, None, scs, 1)


def test_a_scenario_needs_both_node_sets():
    with pytest.raises(ValueError, match="scenario 0 lacks nodesToAdd"):
        blance_b200.PlanNextMapScenarios({}, {}, ["a"], {"primary": (0, 1)}, None, [{"nodesToRemove": []}])


# ---- ABI --------------------------------------------------------------------------------------------------------

def test_scenario_struct_layout_matches_header():
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(blance_scenario), offsetof(blance_scenario, add_is_nil),
             offsetof(blance_scenario, node_weight), sizeof(blance_scenario_out), offsetof(blance_scenario_out, node_ops),
             offsetof(blance_scenario_out, iters_run), offsetof(blance_scenario_out, steps), offsetof(blance_scenario_out, warn_parts));
      return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")], check=True)
        out = list(map(int, subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    S, SO = api.Scenario, api.ScenarioOut
    assert out == [ctypes.sizeof(S), S.add_is_nil.offset, S.node_weight.offset, ctypes.sizeof(SO), SO.node_ops.offset,
                   SO.iters_run.offset, SO.steps.offset, SO.warn_parts.offset]


def _have_gpu():
    lib = api.capi()
    ctx = ctypes.c_void_p()
    st = lib.blance_ctx_create(ctypes.byref(ctx), -1)
    if st == 0:
        lib.blance_ctx_destroy(ctx)
    return st == 0


def test_no_cpu_fallback_for_scenarios():
    if _have_gpu():
        pytest.skip("a CUDA device is present")
    with pytest.raises(blance_b200.BlanceError):
        blance_b200.PlanNextMapScenarios({}, {"0": {}}, ["a"], {"primary": (0, 1)}, None,
                                         [{"nodesToRemove": [], "nodesToAdd": ["a"]}])
