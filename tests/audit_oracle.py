"""A direct reading, over string maps, of the audit that include/blance_b200.h defines ("auditing a partition map"):
plan.go:723-774 (includeExcludeNodes, includeExcludeNodesIntersect, findAncestor, findLeaves on the parent map),
plan.go:134-138 (the top-priority node), plan.go:178-181 (the anchor) and plan.go:228 (the constraints).  It shares
no code with the product: no interning, no bit sets, Go's map and slice semantics spelled out.

    audit(pmap, model, nodes_all, node_hierarchy=None, hierarchy_rules=None, domain_parents=None)

pmap            {partition: {state: [node, ...] | None}}      model   {state: (priority, constraints)}
node_hierarchy  {child: parent} (PlanNextMapOptions.NodeHierarchy), the parent map of the rules
hierarchy_rules {state: [(includeLevel, excludeLevel), ...]}, None = no rules at all
domain_parents  {vertex: parent} of the fault-domain forest, None = every node is its own domain
"""
import collections


def sort_state_names(model):                       # plan.go:437-447: priority ASC, name ASC
    return sorted(model, key=lambda s: (model[s][0], s))


def top_priority_state(model):                     # plan.go:126-132 (ties: the first in state order)
    names = sort_state_names(model)
    return names[0] if names else ""


def map_parents_to_map_children(parents):          # plan.go:703-717
    rv = collections.defaultdict(list)
    for child in sorted(parents):
        rv[parents[child]].append(child)
    return rv


def find_ancestor(node, parents, level):           # plan.go:755-762 (a missing key reads as "")
    while level > 0:
        node = parents.get(node, "")
        level -= 1
    return node


def find_leaves(node, children):                   # plan.go:764-774
    kids = children.get(node, [])
    if len(kids) <= 0:
        return [node]
    rv = []
    for c in kids:
        rv += find_leaves(c, children)
    return rv


def include_exclude_nodes(node, inc, exc, parents, children):      # plan.go:723-734
    inc_nodes = find_leaves(find_ancestor(node, parents, inc), children)
    exc_nodes = set(find_leaves(find_ancestor(node, parents, exc), children))
    return [n for n in inc_nodes if n not in exc_nodes]


def include_exclude_nodes_intersect(nodes, inc, exc, parents, children):   # plan.go:738-753
    rv = []
    for node in nodes:
        res = include_exclude_nodes(node, inc, exc, parents, children)
        if len(rv) == 0:
            rv = res
            continue
        keep = set(res)
        rv = [n for n in rv if n in keep]
    return rv


def _ancestors(v, dparents):
    """v and every vertex above it."""
    out = [v]
    while dparents.get(out[-1]) is not None:
        out.append(dparents[out[-1]])
        assert len(out) <= 17, "forest deeper than 16"
    return out


def audit(pmap, model, nodes_all, node_hierarchy=None, hierarchy_rules=None, domain_parents=None):
    states = sort_state_names(model)
    top = top_priority_state(model)
    parents = node_hierarchy or {}
    children = map_parents_to_map_children(parents)
    dparents = domain_parents or {}
    in_all = set(nodes_all)
    pos = {n: i for i, n in enumerate(nodes_all)}
    C = collections.Counter
    r = dict(short_slots=C(), over_slots=C(), rule_miss=C(), rule_tested=C(), dom_top=C(), dom_all=C(), dom_copies=C(),
             n2n=C(), short_parts=0, rule_miss_parts=0, no_top_parts=0, part_flags={})
    for name, nbs in pmap.items():
        lists = {s: list(nbs[s] or []) for s in states if s in nbs}          # only model states count
        top_nodes = lists.get(top, [])
        h = top_nodes[0] if len(top_nodes) > 0 else ""                        # plan.go:134-138
        short = miss = False
        for s in states:
            k = model[s][1]
            if s not in lists or k <= 0:
                continue
            L = lists[s]
            if len(L) < k:
                r["short_slots"][s] += k - len(L)
                short = True
            if len(L) > k:
                r["over_slots"][s] += len(L) - k
            if hierarchy_rules is None:
                continue
            for ri, (inc, exc) in enumerate(hierarchy_rules.get(s, [])):
                for j in range(min(len(L), k)):
                    if s == top and j == 0:
                        continue
                    a = h
                    if a == "" and j > 0:                                     # plan.go:178-181
                        a = L[0]
                    cand = include_exclude_nodes_intersect([a] + L[:j], inc, exc, parents, children)
                    cand = [n for n in cand if n in in_all]                   # plan.go:193-194
                    r["rule_tested"][(s, ri)] += 1
                    if L[j] not in cand:
                        r["rule_miss"][(s, ri)] += 1
                        miss = True
        copies = [n for s in states for n in lists.get(s, [])]
        for n in copies:
            for v in _ancestors(n, dparents):
                r["dom_copies"][v] += 1
            if h != "" and n != h and n in in_all and h in in_all:
                r["n2n"][(h, n)] += 1
        if h != "":
            for v in _ancestors(h, dparents):
                r["dom_top"][v] += 1
        if copies:
            common = None
            for n in copies:
                anc = _ancestors(n, dparents)
                common = anc if common is None else [v for v in common if v in anc]
            for v in common:
                r["dom_all"][v] += 1
        r["short_parts"] += short
        r["rule_miss_parts"] += miss
        r["no_top_parts"] += h == ""
        r["part_flags"][name] = (1 if short else 0) | (2 if miss else 0) | (4 if h == "" else 0)
    best = (0, None, None)
    for (a, b), c in sorted(r["n2n"].items(), key=lambda kv: (pos[kv[0][0]], pos[kv[0][1]])):
        if c > best[0]:
            best = (c, a, b)
    r["n2n_max"] = best
    for k, v in list(r.items()):
        if isinstance(v, C):
            r[k] = {a: b for a, b in v.items() if b}
    return r
