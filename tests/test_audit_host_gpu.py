"""The string-level audit on the device: AuditMap gives the hand-derived counts of the reference's expected maps
(tests/test_audit_goldens.py) and equals the oracle on them and on random string maps; PlanNextMapScenarios(audit=...)
equals AuditMap of each scenario's final map and changes nothing else.  Needs an H100; run with -m gpu."""
import random

import pytest

import audit_oracle as AO
import golden_util as G
from test_audit_goldens import HAND, hand_cases

import blance_b200

pytestmark = pytest.mark.gpu


def in_oracle_form(a):
    """AuditMap's dict with the oracle's keys."""
    r = {k: a[k] for k in ("short_slots", "over_slots", "dom_top", "dom_all", "dom_copies", "short_parts", "rule_miss_parts", "no_top_parts")}
    for f in ("rule_miss", "rule_tested"):
        r[f] = {(s, i): c for s, v in a[f].items() for i, c in enumerate(v) if c}
    r["part_flags"] = a["part_flags"]
    if "failover_spread" in a:
        r["n2n"] = {(x, y): c for x, v in a["failover_spread"].items() for y, c in v.items()}
        c, x, y = a["failover_max"]
        r["n2n_max"] = (c, x, y) if c else (0, None, None)
    return r


def same(a, o, n2n=True):
    o = dict(o)
    o["part_flags"] = {k: v for k, v in o["part_flags"].items() if v}
    if not n2n:
        o.pop("n2n"), o.pop("n2n_max")
    assert in_oracle_form(a) == o


def options(kw):
    return blance_b200.PlanNextMapOptions(ModelStateConstraints=kw["model_state_constraints"], NodeHierarchy=kw["node_hierarchy"],
                                          HierarchyRules=kw["hierarchy_rules"])


@pytest.mark.parametrize("c", hand_cases(), ids=G.case_id)
def test_audit_map_gives_the_hand_derived_counts(c):
    kw = G.plan_kwargs(c)
    pm = G.pmap(c["exp"])
    a = blance_b200.AuditMap(pm, kw["nodes_all"], kw["model"], options(kw), failoverSpread=True)
    t, m, mp, sh, sp = HAND[(c["group"], c["index"])][1:]
    assert (sum(a["rule_tested"].get("replica", [])), sum(a["rule_miss"].get("replica", [])), a["rule_miss_parts"],
            a["short_slots"].get("replica", 0), a["short_parts"]) == (t, m, mp, sh, sp)
    same(a, AO.audit(pm, kw["model"], kw["nodes_all"], kw["node_hierarchy"], kw["hierarchy_rules"], kw["node_hierarchy"]))


def random_case(seed):
    rnd = random.Random(seed)
    n = rnd.randint(3, 40)
    nodes = ["n%02d" % i for i in range(n)]
    others = ["x%d" % i for i in range(rnd.randint(0, 2))]               # in maps, not in nodesAll
    model = {"primary": (0, rnd.randint(0, 2)), "replica": (1, rnd.randint(0, 3)), "standby": (rnd.choice([1, 2]), rnd.randint(0, 2))}
    f1, f2 = rnd.randint(1, 5), rnd.randint(1, 3)
    nh = {}
    for i, x in enumerate(nodes + others):
        if rnd.random() < 0.9:
            nh[x] = "rack%02d" % (i // f1)
    for r in sorted(set(nh.values())):
        if rnd.random() < 0.9:
            nh[r] = "zone%d" % (int(r[4:]) // f2)
    nh["ghost"] = "rack00"
    rules = {s: [(rnd.randint(0, 3), rnd.randint(0, 2)) for _ in range(rnd.randint(1, 2))] for s in model if rnd.random() < 0.7}
    pm = {}
    for p in range(rnd.randint(1, 300)):
        pool = rnd.sample(nodes + others, min(len(nodes), 8))
        nbs = {}
        for s, (_, k) in model.items():
            u = rnd.random()
            if u < 0.08:
                continue
            nbs[s] = None if u < 0.12 else [pool.pop() for _ in range(min(len(pool), rnd.choice([k, k, k, max(0, k - 1), k + 1])))]
        if rnd.random() < 0.1:
            nbs["unknown"] = [nodes[0]]
        pm["p%04d" % p] = nbs
    return pm, nodes, model, nh, rules


@pytest.mark.parametrize("chunk", range(3))
def test_audit_map_equals_the_oracle_on_random_maps(chunk):
    for seed in range(chunk * 8, chunk * 8 + 8):
        pm, nodes, model, nh, rules = random_case(seed)
        for use_nh, use_rules, n2n in ((True, True, True), (True, False, False), (False, True, True), (False, False, False)):
            o = blance_b200.PlanNextMapOptions(NodeHierarchy=nh if use_nh else None, HierarchyRules=rules if use_rules else None)
            a = blance_b200.AuditMap(pm, nodes, model, o, failoverSpread=n2n)
            same(a, AO.audit(pm, model, nodes, nh if use_nh else None, rules if use_rules else None, nh if use_nh else None), n2n)
    a = blance_b200.AuditMap(pm, nodes, model, blance_b200.PlanNextMapOptions(ModelStateConstraints={"replica": 4}))
    same(a, AO.audit(pm, dict(model, replica=(1, 4)), nodes), False)


def test_bad_hierarchy_is_refused():
    with pytest.raises(blance_b200.BlanceError, match="cycle"):
        blance_b200.AuditMap({"p": {"primary": ["a"]}}, ["a"], {"primary": (0, 1)},
                             blance_b200.PlanNextMapOptions(NodeHierarchy={"a": "r", "r": "q", "q": "r"}))


def test_scenarios_audit_equals_audit_map_of_each_final_map():
    c = next(c for c in hand_cases() if c["index"] == 0 and "MultiRack" in c["group"])        # 3 racks of 3 nodes, k = 2
    kw = G.plan_kwargs(c)
    prev = G.pmap(c["exp"])
    o = options(kw)
    scs = [{"nodesToRemove": rm, "nodesToAdd": None} for rm in ([], ["a", "b", "c"], ["a", "b", "c", "d", "e", "f"], ["e"])]
    scs.append({"nodesToRemove": ["g"], "nodesToAdd": None, "modelStateConstraints": {"replica": 1}})
    scs.append({"nodesToRemove": ["g"], "nodesToAdd": None, "hierarchyRules": {"replica": [(1, 0)]}})
    plain = blance_b200.PlanNextMapScenarios(prev, prev, kw["nodes_all"], kw["model"], o, scs, wantMaps=range(len(scs)), scheduleConcurrency=[1])
    res = blance_b200.PlanNextMapScenarios(prev, prev, kw["nodes_all"], kw["model"], o, scs, wantMaps=range(len(scs)), scheduleConcurrency=[1],
                                           audit={"failoverSpread": True})
    assert all("audit" not in d for d in plain)
    assert [{k: v for k, v in d.items() if k != "audit"} for d in res] == plain
    for sc, d in zip(scs, res):
        final = dict(prev)
        final.update(d["next_map"])
        so = blance_b200.PlanNextMapOptions(ModelStateConstraints=sc.get("modelStateConstraints"), NodeHierarchy=kw["node_hierarchy"],
                                            HierarchyRules=sc.get("hierarchyRules", kw["hierarchy_rules"]))
        assert d["audit"] == blance_b200.AuditMap(final, kw["nodes_all"], kw["model"], so, failoverSpread=True)
    # two racks gone: every replica sits in its primary's rack and the planner warned about nothing
    assert res[2]["warn_parts"] == 0 and res[2]["audit"]["rule_miss_parts"] == len(prev)
    assert res[0]["audit"]["rule_miss_parts"] == 0
    no_sched = blance_b200.PlanNextMapScenarios(prev, prev, kw["nodes_all"], kw["model"], o, scs, audit={})
    assert all("schedules" not in d and "failover_max" not in d["audit"] for d in no_sched)
    assert [d["audit"]["rule_miss"] for d in no_sched] == [d["audit"]["rule_miss"] for d in res]
