"""The audit oracle (tests/audit_oracle.py) on cases derived by hand from plan.go:723-774, 134-138 and 178-181, and
the interning the audit tests rely on (the fault-domain forest and the hierarchy bit sets of tests/audit_util.py).
No device."""
import numpy as np

import audit_oracle as AO
import audit_util as U
from blance_b200 import tables

# two racks of two nodes in one zone; e's rack r2 has no zone; f is outside the hierarchy
PARENTS = {"a": "r0", "b": "r0", "c": "r1", "d": "r1", "r0": "z0", "r1": "z0", "e": "r2"}
NODES = ["a", "b", "c", "d", "e", "f"]
RULES = {"replica": [(2, 1)]}          # same zone, another rack


def audit(pmap, k_replica=2, rules=RULES, **kw):
    return AO.audit(pmap, {"primary": (0, 1), "replica": (1, k_replica)}, NODES, PARENTS, rules, **kw)


def test_second_replica_of_two_racks_cannot_comply():
    # j = 0: [a] -> {c, d}, c complies.  j = 1: [a, c] -> {c, d} & {a, b} = {}: d misses (plan.go:750), which is
    # where findBestNodes falls back to the flat best node (plan.go:214-220)
    r = audit({"p": {"primary": ["a"], "replica": ["c", "d"]}})
    assert r["rule_tested"] == {("replica", 0): 2} and r["rule_miss"] == {("replica", 0): 1}
    assert r["rule_miss_parts"] == 1 and r["short_parts"] == 0 and r["part_flags"] == {"p": 2}


def test_replace_on_empty():
    # [a, c] leaves rv empty, so b REPLACES it (plan.go:746-749): [a, c, b] -> {c, d} and d complies at j = 2
    r = audit({"p": {"primary": ["a"], "replica": ["c", "b", "d"]}}, k_replica=3)
    assert r["rule_tested"] == {("replica", 0): 3} and r["rule_miss"] == {("replica", 0): 1}


def test_empty_anchor():
    # no primary: h = "" (plan.go:134-138).  j = 0: [""] -> leaves("") minus leaves("") = {}: a misses.
    # j = 1: the anchor is L[0] = a (plan.go:178-181): [a, a] -> {c, d}: c complies
    r = audit({"p": {"replica": ["a", "c"]}})
    assert r["rule_tested"] == {("replica", 0): 2} and r["rule_miss"] == {("replica", 0): 1}
    assert r["no_top_parts"] == 1 and r["part_flags"] == {"p": 2 | 4} and r["dom_top"] == {}


def test_missing_ancestor_keeps_the_set_non_empty():
    # e's level-2 ancestor is "" (control_test.go:373-384): leaves("") = [""], minus leaves(r2) = [e] -> [""], a set
    # that is NOT empty.  So [e, c] -> [""] & {a, b} = {}: a misses; had "" been dropped, c would have replaced the
    # set and a would comply
    r = audit({"p": {"primary": ["e"], "replica": ["c", "a"]}})
    assert r["rule_miss"] == {("replica", 0): 2}


def test_node_outside_the_hierarchy():
    # f has no parent: both ancestors are "", the set is empty, c misses; f is its own fault domain
    dp = {k: v for k, v in PARENTS.items()}
    r = audit({"p": {"primary": ["f"], "replica": ["c"]}}, k_replica=1, domain_parents=dp)
    assert r["rule_miss"] == {("replica", 0): 1}
    assert r["dom_copies"] == {"f": 1, "c": 1, "r1": 1, "z0": 1} and r["dom_top"] == {"f": 1} and r["dom_all"] == {}


def test_constraints_domains_and_failover_spread():
    pmap = {"p0": {"primary": ["a"], "replica": ["b"]},                 # one replica short; both copies in r0
            "p1": {"primary": ["a"], "replica": ["c", "d", "b"]},       # one over
            "p2": {"primary": None, "replica": None},                   # lists present and empty
            "p3": {"other": ["a"]}}                                     # no model state at all
    r = audit(pmap, rules=None, domain_parents=PARENTS)
    assert r["short_slots"] == {"primary": 1, "replica": 1 + 2} and r["over_slots"] == {"replica": 1}
    assert r["short_parts"] == 2 and r["no_top_parts"] == 2
    assert r["dom_top"] == {"a": 2, "r0": 2, "z0": 2}
    assert r["dom_all"] == {"r0": 1, "z0": 2}
    assert r["dom_copies"] == {"a": 2, "b": 2, "c": 1, "d": 1, "r0": 4, "r1": 2, "z0": 6}
    assert r["n2n"] == {("a", "b"): 2, ("a", "c"): 1, ("a", "d"): 1} and r["n2n_max"] == (2, "a", "b")
    assert r["part_flags"] == {"p0": 1, "p1": 0, "p2": 1 | 4, "p3": 4}
    assert r["rule_tested"] == {}


def test_interning_of_the_test_helpers():
    t = tables.PlanTables(4, 2, 1, [0, 1], [1, 2], n_node_ids=5)
    names = ["a", "b", "c", "d", "e"]
    arr, vnames = U.forest(t, PARENTS, names)
    assert vnames == names + ["r0", "r1", "r2", "z0"]
    assert arr.tolist() == [5, 5, 6, 6, 7, 8, 8, -1, -1]
    U.set_hierarchy(t, PARENTS, {"s1": [(2, 1)]}, names)
    mask = np.asarray(t.ie_mask).reshape(1, 6, t.hier_words)
    assert t.n_rules == 1 and t.rule_off.tolist() == [0, 0, 1] and t.n_hier_bits == 5         # one extra leaf: ""
    assert mask[0, :, 0].tolist() == [0b1100, 0b1100, 0b0011, 0b0011, 0b10000, 0]
