"""The audit of the reference's own expected maps (tests/golden/plan_cases.json), every count derived by hand from
the Vis rows of plan_test.go / control_test.go and written here with the line the case starts at.  The oracle
(tests/audit_oracle.py) must give these numbers (no device); tests/test_audit_host_gpu.py holds the product to them.

All rules are on "replica"; T = tested positions, M = misses, MP = partitions with a miss, SH = replica slots short,
SP = partitions short.  How each was derived:

 plan_test.go:2267  rule (1,0) "same rack, not itself": every replica shares its primary's rack          T 8  M 0
 plan_test.go:2288  rule (2,1) "same zone, other rack"; pairs a-c b-d c-a d-b a-d b-c c-b d-a all cross   T 8  M 0
 plan_test.go:2309  e-a b-e c-a d-b a-d b-c c-b d-a, e is in r1: all cross                                 T 8  M 0
 plan_test.go:2332  a-c a-d c-a d-a a-d c-a c-a d-a: all cross                                             T 8  M 0
 plan_test.go:2653  3 racks, k = 2: position 0 is outside the primary's rack in all 8 rows; position 1 must be in the
                    third rack ([p, r0] excludes two racks): a|i,d  b|e,g  c|f,h  d|i,a  e|b,g  f|c,h  g|a,d  h|b,e
                    - the second replica is in the remaining rack every time                               T 16 M 0
 plan_test.go:2675  only rack r0 is left, k = 2: both replicas of all 8 rows sit in the primary's rack; the set for
                    position 1 is {d..i} & {d..i}, still without r0                                        T 16 M 16 MP 8
 plan_test.go:2697  4 racks of one node, k = 3: a|b,c,d -> {b,c,d}, {c,d}, {d}; b|a,c,d; c|a,b,d -> {a,b,d}, {b,d},
                    {d}; d|a,b,c -> {a,b,c}, {b,c}, {c}: every position complies                           T 12 M 0
 plan_test.go:2731  the 4-warning case: a and e (both r0) are left, k = 3, each row has ONE replica, in the primary's
                    rack: 1 tested and missed per row, 2 slots short per row                               T 4  M 4  MP 4  SH 8  SP 4
 plan_test.go:2766  a-c b-d c-a d-b                                                                        T 4  M 0
 plan_test.go:2798  rack r0 is down: c-d d-c c-d d-c, all inside r1, and no warning                        T 4  M 4  MP 4
 plan_test.go:2830  one rack: a-b b-a c-a a-c b-c c-b                                                      T 6  M 6  MP 6
 control_test.go:309 groups without a parent: the level-2 ancestor of a is "" (control_test.go:373-384), the set is
                    [""], b is not in it; likewise for Y                                                   T 2  M 2  MP 2
"""
import pytest

import audit_oracle as AO
import golden_util as G

#        group, index                                           line   T   M  MP  SH  SP
HAND = {("TestPlanNextMapHierarchy", 1): (2267, 8, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchy", 2): (2288, 8, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchy", 3): (2309, 8, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchy", 4): (2332, 8, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 0): (2653, 16, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 1): (2675, 16, 16, 8, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 2): (2697, 12, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 3): (2731, 4, 4, 4, 8, 4),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 4): (2766, 4, 0, 0, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 5): (2798, 4, 4, 4, 0, 0),
        ("TestPlanNextMapHierarchyMultiRackFailureCases", 6): (2830, 6, 6, 6, 0, 0),
        ("TestControlCase4", 0): (309, 2, 2, 2, 0, 0)}


def hand_cases():
    cs = [c for c in G.plan_cases() if (c["group"], c["index"]) in HAND]
    assert len(cs) == len(HAND)
    return cs


def as_counts(r):
    """(T, M, MP, SH, SP) of an audit in the oracle's form."""
    assert set(r["rule_tested"]) <= {("replica", 0)} and set(r["short_slots"]) <= {"replica"} and not r["over_slots"]
    return (r["rule_tested"].get(("replica", 0), 0), r["rule_miss"].get(("replica", 0), 0), r["rule_miss_parts"],
            r["short_slots"].get("replica", 0), r["short_parts"])


@pytest.mark.parametrize("c", hand_cases(), ids=G.case_id)
def test_oracle_gives_the_hand_derived_counts(c):
    kw = G.plan_kwargs(c)
    r = AO.audit(G.pmap(c["exp"]), kw["model"], kw["nodes_all"], kw["node_hierarchy"], kw["hierarchy_rules"], kw["node_hierarchy"])
    assert as_counts(r) == HAND[(c["group"], c["index"])][1:]
    assert r["no_top_parts"] == 0
    # what the planner itself reported: warnings only where slots are short, none for the misses
    assert (c["expNumWarnings"] > 0) == (r["short_parts"] > 0)


def test_interning_of_the_fault_domain_forest():
    """AuditMap's forest: node ids first (nodesAll, then other names of the map), then the hierarchy's other names in
    byte order; a node outside the hierarchy and a name whose parent is "" are roots."""
    import blance_b200
    from blance_b200 import _host
    pm = {"p": {"primary": ["b"], "replica": ["x", "a"]}}
    ip = _host.intern_plan(pm, None, ["a", "b", "c"], None, None, {"primary": (0, 1), "replica": (1, 2)})
    assert ip.node_names == ["a", "b", "c", "x"]
    nh = {"a": "r1", "b": "r0", "r0": "z", "r1": "z", "z": "", "ghost": "r0"}
    names, parent = _host.audit_forest(ip, nh)
    assert names == ["a", "b", "c", "x", "ghost", "r0", "r1", "z"]
    assert parent == [6, 5, -1, -1, 5, 7, 7, -1]
    assert _host.audit_forest(ip, None) == (["a", "b", "c", "x"], [])
    assert blance_b200.AuditMap is not None
