"""What-if scenarios that vary plan options (ModelStateConstraints, StateStickiness, PartitionWeights, NodeHierarchy,
HierarchyRules), CPU side: each scenario's substituted tables (InternScenario) planned by the table oracle equal the
literal oracle on the string-level inputs with those options substituted; the blance_scenario_opts layout; and the
host layer's input checks.  No device needed (the device path is tests/test_scenario_options_gpu.py)."""
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
from blance_b200 import _host, abi, api

L = literal()
FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# scenario key -> PlanNextMapEx keyword of the literal oracle
OPTION_KEYS = {"nodeWeights": "node_weights", "modelStateConstraints": "model_state_constraints",
               "stateStickiness": "state_stickiness", "partitionWeights": "partition_weights",
               "nodeHierarchy": "node_hierarchy", "hierarchyRules": "hierarchy_rules"}


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
    for key, arg in OPTION_KEYS.items():
        if key in sc:
            k[arg] = copy.deepcopy(sc[key])
    return k


def constraints_of(kw):
    msc = kw.get("model_state_constraints") or {}
    return {s: msc.get(s, k) for s, (_p, k) in kw["model"].items()}


def rules_fit(kw, constraints, rules):
    """The device's limit of hierarchy picks per step: rules x constraints <= 32 for every state."""
    rules = rules or {}
    return all(len(rules.get(s, ())) * max(0, k) <= 32 for s, k in constraints.items())


def extra_state_partition(kw):
    """A prevMap partition that also holds a state outside the model (it feeds the non-model counts)."""
    for p, nbs in sorted(kw["prev_map"].items()):
        if any(s not in kw["model"] for s in nbs):
            return p
    return None


def make_option_scenarios(kw, seed, all_states=True):
    """Option variants of one case, each with the case's own node sets: constraints +-1 per state within the
    limits, stickiness {0, 1, 3} (cases with PartitionWeights), PartitionWeights nil / inherited / changed
    (including a partition holding non-model states), hierarchy rules dropped or added, a node moved to another
    parent."""
    own = {"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": kw["nodes_to_add"]}
    scs = [dict(own)]
    cons = constraints_of(kw)
    states = sorted(cons)
    for i, s in enumerate(states):
        if not all_states and i != seed % len(states):
            continue
        for d in (1, -1):
            k = cons[s] + d
            if 0 <= k <= 16:
                c = dict(cons)
                c[s] = k
                if rules_fit(kw, c, kw.get("hierarchy_rules")):
                    scs.append(dict(own, modelStateConstraints=c))
    pw = kw.get("partition_weights")
    if pw is not None:
        for v in (0, 1, 3):
            scs.append(dict(own, stateStickiness={s: v for s in states}))
    scs.append(dict(own, partitionWeights=None))
    parts = sorted(set(kw["prev_map"]) | set(kw["partitions_to_assign"] or {}))
    if parts:
        w = dict(pw or {})
        for p in parts[seed % len(parts)::3][:3]:
            w[p] = w.get(p, 1) * 4 + 1
        ex = extra_state_partition(kw)
        if ex is not None:
            w[ex] = 7
        w["zz-not-a-partition"] = 5                     # names outside the maps are ignored
        scs.append(dict(own, partitionWeights=w))
        if pw:
            dropped = dict(pw)
            dropped.pop(sorted(pw)[0])
            scs.append(dict(own, partitionWeights=dropped))
    rules = kw.get("hierarchy_rules")
    nh = kw.get("node_hierarchy")
    if rules is not None:
        scs.append(dict(own, hierarchyRules=None))
    top = min(states, key=lambda s: (kw["model"][s][0], s)) if states else None
    other = [s for s in states if s != top]
    if other:
        added = dict(rules or {})
        added[other[0]] = [(2, 1)] if nh else [(1, 0)]
        if rules_fit(kw, cons, added):
            scs.append(dict(own, hierarchyRules=added))
    if nh:
        leaves = sorted(k for k in nh if k in kw["nodes_all"])
        parents = sorted(set(nh.values()))
        if leaves and len(parents) > 1:
            moved = dict(nh)
            q = leaves[seed % len(leaves)]
            moved[q] = [x for x in parents if x != nh[q]][0]
            scs.append(dict(own, nodeHierarchy=moved))
    return scs


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
        assert next_map == lit["next_map"], (i, sc)
        assert warnings == lit["warnings"], (i, sc)
        assert out.iters_run == lit["iterations"], (i, sc)


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_option_scenarios_match_literal_oracle_golden(c):
    kw = G.plan_kwargs(c)
    check_scenarios(kw, make_option_scenarios(kw, c["index"]))


@pytest.mark.parametrize("chunk", range(6))
def test_option_scenarios_match_literal_oracle_random(chunk):
    for seed in range(chunk * 50, (chunk + 1) * 50):
        kw = random_instance(seed)
        check_scenarios(kw, make_option_scenarios(kw, seed, all_states=False))


def test_raised_constraints_widen_the_shared_layout():
    """A scenario that raises a constraint widens every scenario's slot range; the base still plans as before."""
    kw = G.plan_kwargs(G.plan_cases()[0])
    cons = constraints_of(kw)
    s = sorted(cons)[0]
    up = dict(cons)
    up[s] = cons[s] + 2
    own = {"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": kw["nodes_to_add"]}
    scs = [dict(own), dict(own, modelStateConstraints=up)]
    o = options_of(kw)
    assign = kw["prev_map"] if kw["partitions_to_assign"] is None else kw["partitions_to_assign"]
    alone = api.intern_scenario(kw["prev_map"], assign, kw["nodes_all"], kw["model"], o, scs[:1], 0)
    wide = api.intern_scenario(kw["prev_map"], assign, kw["nodes_all"], kw["model"], o, scs, 0)
    assert wide.n_slots == alone.n_slots + 2
    assert list(wide.tables()["state_constraints"]) == list(alone.tables()["state_constraints"])
    check_scenarios(kw, scs)


def test_weight_overrides_are_the_difference_to_the_base():
    prev = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}, "2": {"primary": ["a"], "dead": ["b"]}}
    model = {"primary": (0, 1)}
    o = blance_b200.PlanNextMapOptions(PartitionWeights={"0": 2, "1": 3})
    own = {"nodesToRemove": [], "nodesToAdd": []}
    scs = [dict(own), dict(own, partitionWeights={"0": 2, "2": 9}), dict(own, partitionWeights=None)]
    assign = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}}
    t = [api.intern_scenario(prev, assign, ["a", "b"], model, o, scs, i).tables() for i in range(3)]
    assert list(t[0]["part_weight"]) == [2, 3, 1]
    assert list(t[1]["part_weight"]) == [2, 1, 9]        # "1" lost its weight, "2" gained one
    assert list(t[2]["part_weight"]) == [2, 3, 1]        # nil: the flags are not read, nothing to override


# ---- invalid input ----------------------------------------------------------------------------------------------

def test_constraints_beyond_the_limit_name_the_scenario():
    prev = {"0": {"primary": ["a"]}}
    own = {"nodesToRemove": [], "nodesToAdd": None}
    scs = [dict(own), dict(own, modelStateConstraints={"primary": 17})]
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: constraints 17"):
        blance_b200.PlanNextMapScenarios(prev, prev, ["a", "b"], {"primary": (0, 1)}, None, scs)
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: constraints 17"):
        api.intern_scenario(prev, prev, ["a", "b"], {"primary": (0, 1)}, None, scs, 1)


def test_a_bad_weight_override_names_the_scenario():
    prev = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}}
    own = {"nodesToRemove": [], "nodesToAdd": None}
    scs = [dict(own), dict(own), dict(own, partitionWeights={"1": 1000000000})]
    with pytest.raises(blance_b200.BlanceError, match="scenario 2: partition weight of '1'"):
        blance_b200.PlanNextMapScenarios(prev, prev, ["a", "b"], {"primary": (0, 1)}, None, scs)
    with pytest.raises(blance_b200.BlanceError, match="scenario 2: partition weight of '1'"):
        api.intern_scenario(prev, prev, ["a", "b"], {"primary": (0, 1)}, None, scs, 2)


# ---- ABI --------------------------------------------------------------------------------------------------------

def test_scenario_opts_layout_matches_header():
    fields = [f for f, _ in api.ScenarioOpts._fields_]
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    int main(void) {
      printf("%zu", sizeof(blance_scenario_opts));
      FIELDS
      printf(" %d %d %d %d\n", BLANCE_OPT_CONSTRAINTS, BLANCE_OPT_STICKINESS, BLANCE_OPT_PART_WEIGHTS, BLANCE_OPT_HIERARCHY);
      return 0; }
    '''.replace("FIELDS", "\n".join('printf(" %%zu", offsetof(blance_scenario_opts, %s));' % f for f in fields))
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")], check=True)
        out = list(map(int, subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    O = api.ScenarioOpts
    assert out == ([ctypes.sizeof(O)] + [getattr(O, f).offset for f in fields] +
                   [abi.OPT_CONSTRAINTS, abi.OPT_STICKINESS, abi.OPT_PART_WEIGHTS,
                    abi.OPT_HIERARCHY])
