"""Helpers of the audit tests: random audited instances in flat AND string form, built without the product's
interning (names, the hierarchy bit sets and the fault-domain forest are made here from the oracle's own set
functions), and the oracle's answer turned into arrays over those ids."""
import numpy as np

import audit_oracle as AO
from blance_b200 import tables


def node_names(t):
    return ["n%04d" % i for i in range(t.n_nodes)] + ["x%d" % i for i in range(t.n_node_ids - t.n_nodes)]


def state_names(t):
    return ["s%d" % s for s in range(t.n_states)]           # priority = index: the state order is the index order


def string_map(t, rows, shape, names=None):
    names = names or node_names(t)
    states = state_names(t)
    rows = np.asarray(rows).reshape(t.n_parts, -1)
    shape = np.asarray(shape).reshape(t.n_parts, -1)
    m = {}
    for p in range(t.n_parts):
        nbs = {}
        for s in range(t.n_states):
            if shape[p, s] == 0:
                continue
            lo, hi = int(t.state_slot_off[s]), int(t.state_slot_off[s + 1])
            nodes = []
            for x in rows[p, lo:hi]:
                if x < 0:
                    break
                nodes.append(names[x])
            nbs[states[s]] = None if shape[p, s] == 1 else nodes
        m["p%07d" % p] = nbs
    return m


def model_of(t):
    return {n: (int(t.state_priority[s]), int(t.state_constraints[s])) for s, n in enumerate(state_names(t))}


def set_hierarchy(t, parents, rules_by_state, names=None):
    """Installs the rules on `t` as bit sets built from the oracle's includeExcludeNodes: bits < n_nodes are node
    ids, leaf names outside nodesAll get the bits after them."""
    names = names or node_names(t)
    children = AO.map_parents_to_map_children(parents)
    rules, rule_off = [], [0]
    for s in state_names(t):
        rules += list(rules_by_state.get(s, []))
        rule_off.append(len(rules))
    ids = {n: i for i, n in enumerate(names[:t.n_nodes])}
    extra = {}
    lists = []
    for inc, exc in rules:
        for a in names + [""]:
            bits = []
            for leaf in AO.include_exclude_nodes(a, inc, exc, parents, children):
                bits.append(ids[leaf] if leaf in ids else t.n_nodes + extra.setdefault(leaf, len(extra)))
            lists.append(bits)
    t.has_hier_rules, t.n_rules, t.n_hier_bits = 1, len(rules), t.n_nodes + len(extra)
    t.rule_off = np.asarray(rule_off, np.int32)
    mask = np.zeros((len(lists), t.hier_words), np.uint32)
    for i, bits in enumerate(lists):
        for b in bits:
            mask[i, b >> 5] |= np.uint32(1 << (b & 31))
    t.ie_mask = mask.reshape(-1)


def forest(t, dparents, names=None):
    """(domain_parent array, vertex names): the node ids first, then the inner vertices in first-appearance order."""
    names = list(names or node_names(t))
    vid = {n: i for i, n in enumerate(names)}
    for c in sorted(dparents):
        for v in (c, dparents[c]):
            if v not in vid:
                vid[v] = len(names)
                names.append(v)
    arr = np.full(len(names), -1, np.int32)
    for c, p in dparents.items():
        arr[vid[c]] = vid[p]
    return arr, names


def random_instance(seed, N=None, P=None):
    rng = np.random.default_rng(seed)
    N = N or int(rng.integers(3, 40))
    extra = int(rng.integers(0, 3))
    S = int(rng.integers(1, 4))
    ks = [int(rng.integers(0, 5)) for _ in range(S)]
    if sum(ks) == 0:
        ks[0] = 1
    P = P or int(rng.integers(1, 400))
    t = tables.PlanTables(N, S, P, list(range(S)), ks, n_node_ids=N + extra)
    widths = [k + int(rng.integers(0, 3)) for k in ks]
    t.state_slot_off = np.concatenate([[0], np.cumsum(widths)]).astype(np.int32)
    t.n_slots = int(t.state_slot_off[-1])
    rows = np.full((P, t.n_slots), -1, np.int32)
    shape = np.zeros((P, S), np.uint8)
    for p in range(P):
        pool = rng.permutation(N + extra) if rng.random() < 0.9 else rng.integers(0, N + extra, 64)
        used = 0
        for s in range(S):
            u = rng.random()
            shape[p, s] = 0 if u < 0.08 else 1 if u < 0.12 else 2
            if shape[p, s] != 2:
                continue
            n = int(rng.integers(0, widths[s] + 1)) if rng.random() < 0.4 else min(widths[s], ks[s])
            n = min(n, len(pool) - used)
            rows[p, t.state_slot_off[s]:t.state_slot_off[s] + n] = pool[used:used + n]
            used += n
    t.prev_rows = t.cur_rows = rows
    t.prev_shape = t.cur_shape = shape
    names = node_names(t)
    # a 3-level hierarchy over most names (some nodes stay outside it), with a few leaves no map knows
    f1, f2 = int(rng.integers(1, 6)), int(rng.integers(1, 4))
    parents = {}
    for i, n in enumerate(names):
        if rng.random() < 0.9:
            parents[n] = "rack%d" % (i // f1)
    for r in sorted(set(parents.values())):
        parents[r] = "zone%d" % (int(r[4:]) // f2)
    for z in sorted(v for v in set(parents.values()) if v.startswith("zone")):
        if rng.random() < 0.8:
            parents[z] = "root"
    for g in range(int(rng.integers(0, 3))):
        parents["ghost%d" % g] = "rack%d" % int(rng.integers(0, max(1, (len(names) + f1 - 1) // f1)))
    rules = {}
    for s, n in enumerate(state_names(t)):
        if ks[s] and rng.random() < 0.8:
            cnt = max(1, min(int(rng.integers(1, 3)), 32 // max(1, ks[s])))
            rules[n] = [(int(rng.integers(0, 4)), int(rng.integers(0, 3))) for _ in range(cnt)]
    return dict(t=t, rows=rows, shape=shape, names=names, parents=parents, rules=rules, rng=rng)


def expected(t, o, names, vertex_names=None, part_names=None):
    """The oracle's dict `o` as arrays over t's ids (the order of AuditResult's fields)."""
    states = state_names(t)
    vertex_names = vertex_names or names
    vid = {n: i for i, n in enumerate(vertex_names)}
    nid = {n: i for i, n in enumerate(names)}
    R = int(t.n_rules) if t.has_hier_rules else 0
    rule_index = {}
    for s, n in enumerate(states):
        for k in range(int(t.rule_off[s + 1] - t.rule_off[s]) if R else 0):
            rule_index[(n, k)] = int(t.rule_off[s]) + k
    e = dict(short_slots=np.zeros(t.n_states, np.int64), over_slots=np.zeros(t.n_states, np.int64),
             rule_miss=np.zeros(R, np.int64), rule_tested=np.zeros(R, np.int64))
    for f in ("short_slots", "over_slots"):
        for n, c in o[f].items():
            e[f][states.index(n)] = c
    for f in ("rule_miss", "rule_tested"):
        for key, c in o[f].items():
            e[f][rule_index[key]] = c
    for f in ("dom_top", "dom_all", "dom_copies"):
        e[f] = np.zeros(len(vertex_names), np.int64)
        for v, c in o[f].items():
            e[f][vid[v]] = c
    e["n2n"] = np.zeros((t.n_nodes, t.n_nodes), np.int32)
    for (a, b), c in o["n2n"].items():
        e["n2n"][nid[a], nid[b]] = c
    c, a, b = o["n2n_max"]
    e["n2n_max"] = (c, nid[a], nid[b]) if c else (0, -1, -1)
    part_names = part_names or sorted(o["part_flags"])
    e["part_flags"] = np.asarray([o["part_flags"][p] for p in part_names], np.uint8)
    for f in ("short_parts", "rule_miss_parts", "no_top_parts"):
        e[f] = int(o[f])
    return e


def assert_audit(got, e, n2n, what=""):
    for f in ("short_slots", "over_slots", "rule_miss", "rule_tested", "dom_top", "dom_all", "dom_copies", "part_flags"):
        assert np.array_equal(getattr(got, f), e[f]), (what, f, getattr(got, f), e[f])
    for f in ("short_parts", "rule_miss_parts", "no_top_parts"):
        assert getattr(got, f) == e[f], (what, f, getattr(got, f), e[f])
    if n2n:
        assert np.array_equal(got.n2n, e["n2n"]), (what, "n2n")
        assert got.n2n_max == e["n2n_max"], (what, got.n2n_max, e["n2n_max"])
    else:
        assert got.n2n_max == (-1, -1, -1), (what, got.n2n_max)


def oracle_of(t, rows, shape, names, parents=None, rules=None, dparents=None):
    return AO.audit(string_map(t, rows, shape, names), model_of(t), names[:t.n_nodes], parents,
                    rules if t.has_hier_rules else None, dparents)
