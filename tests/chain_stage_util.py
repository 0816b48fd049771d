"""Chains whose stages set plan options of their own (blance_plan_chains_ex), CPU side: the per-stage form of
chain_util.chain_reference, per-stage option sequences of a case, the chain in table form with each stage's options
as an option dict, and the literal oracle driven as the Go loop with per-stage options on string maps."""
import copy
import random

import numpy as np

import chain_util as C
from oracle_loader import literal
from test_scenario_options import OPTION_KEYS, constraints_of, options_of, rules_fit
from test_scenarios_gpu import reference_summary

from blance_b200 import abi, api

L = literal()


def chain_reference_staged(base, chain, stage_opts=None, favor_min_nodes=False):
    """chain_util.chain_reference with stage t planned under stage_opts[t] (a dict of OPT_GROUPS keys, None = the
    base's options) instead of one dict for every stage.  The net summary's moves do not depend on the options."""
    cur, out = base, []
    for t, stage in enumerate(chain):
        x = C.substituted(cur, stage, None if stage_opts is None else stage_opts[t], t)
        r, order = C.renumbered(x, stage.get("node_in_all"))
        ref = C.oracle(r)
        nxt = np.where(ref.next_rows >= 0, order[np.maximum(ref.next_rows, 0)], -1).astype(np.int32)
        res = dict(next_rows=nxt, next_shape=ref.next_shape.copy(), warn=ref.warn.copy(), iters_run=ref.iters_run,
                   converged=ref.converged, steps=ref.steps)
        res.update(reference_summary(x, nxt, ref.warn, favor_min_nodes))
        out.append(res)
        cur = C.advance(cur, nxt, ref.next_shape)
    last = None if stage_opts is None else stage_opts[-1]
    s = reference_summary(C.substituted(base, chain[-1], last, 0), out[-1]["next_rows"], out[-1]["warn"], favor_min_nodes)
    return out, dict(node_ops=s["node_ops"], ops_total=s["ops_total"], parts_moved=s["parts_moved"])


def make_stage_options(kw, seed, T):
    """Per-stage option keys (scenario form) for a T-stage chain of case kw, one pattern per seed: a constraint raised
    at stage 1 and back to the base's after it; stickiness changed at one stage; partition weights changed at stage 0
    (a weight dropped, one added, one changed) and back to the base's at stage 1, nil at stage 2; hierarchy rules
    switched off at stage 0 and first switched on, with a rule more, at the last stage."""
    rnd = random.Random(seed * 17 + 3)
    out = [dict() for _ in range(T)]
    cons = constraints_of(kw)
    states = sorted(cons)
    if not states:
        return out
    pw, rules, nh = kw.get("partition_weights"), kw.get("hierarchy_rules"), kw.get("node_hierarchy")
    kind = seed % 4
    if kind == 1 and pw is None:
        kind = 0
    if kind == 0:
        s = states[seed % len(states)]
        c = dict(cons)
        c[s] = cons[s] + 1
        if c[s] <= 16 and rules_fit(kw, c, rules):
            out[min(1, T - 1)]["modelStateConstraints"] = c
    elif kind == 1:
        out[rnd.randrange(T)]["stateStickiness"] = {s: rnd.choice([0, 1, 3]) for s in states}
    elif kind == 2:
        parts = sorted(set(kw["prev_map"]) | set(kw["partitions_to_assign"] or {}))
        w = dict(pw or {})
        if w:
            w.pop(sorted(w)[seed % len(w)])
        for p in parts[seed % max(1, len(parts))::2][:3]:
            w[p] = w.get(p, 1) * 3 + 2
        out[0]["partitionWeights"] = w
        if T > 2:
            out[2]["partitionWeights"] = None
    else:
        top = min(states, key=lambda s: (kw["model"][s][0], s))
        other = [s for s in states if s != top]
        out[0]["hierarchyRules"] = None
        if other:
            later = dict(rules or {})
            later[other[0]] = list(later.get(other[0], [])) + ([(2, 1)] if nh else [(1, 0)])
            if rules_fit(kw, cons, later):
                out[T - 1]["hierarchyRules"] = later
    return out


def literal_chain_staged(kw, stages, stage_keys):
    """The Go host loop on string maps with the literal oracle; stage t's options are kw's with stage_keys[t]
    substituted (a stage's options do not carry over to the next)."""
    prev = copy.deepcopy(kw["prev_map"])
    assign = copy.deepcopy(kw["partitions_to_assign"])
    out = []
    for (nodes_all, rm, add, nw), keys in zip(stages, stage_keys):
        k = copy.deepcopy(kw)
        k.update(prev_map=copy.deepcopy(prev), partitions_to_assign=copy.deepcopy(assign), nodes_all=list(nodes_all),
                 nodes_to_remove=copy.deepcopy(rm), nodes_to_add=copy.deepcopy(add))
        if nw != "inherit":
            k["node_weights"] = copy.deepcopy(nw)
        for key, v in keys.items():
            k[OPTION_KEYS[key]] = copy.deepcopy(v)
        lit = L.plan_next_map_ex(**k)
        out.append(lit)
        nxt = lit["next_map"]
        prev = dict(prev)
        prev.update(copy.deepcopy(nxt))
        assign = copy.deepcopy(nxt)
    return out


def option_dict(x, base):
    """Every option group of tables x (a stage interned with its options) as an option dict over base: weights as
    overrides of the partitions whose weight or presence differ from the base's."""
    pw, ph = np.asarray(x.part_weight, np.int32), np.asarray(x.part_has_weight, np.uint8)
    part = np.flatnonzero((pw != np.asarray(base.part_weight)) | (ph != np.asarray(base.part_has_weight))).astype(np.int32)
    return dict(state_constraints=np.array(x.state_constraints, np.int32), state_stickiness=np.array(x.state_stickiness, np.int32),
                state_has_stickiness=np.array(x.state_has_stickiness, np.uint8), has_part_weights=int(x.has_part_weights),
                weight_overrides=(part, pw[part], ph[part]), extra_tot_first=np.array(x.extra_tot_first, np.int32),
                extra_tot_rest=np.array(x.extra_tot_rest, np.int32), has_hier_rules=int(x.has_hier_rules),
                n_rules=int(x.n_rules), n_hier_bits=int(x.n_hier_bits), rule_off=np.array(x.rule_off, np.int32),
                ie_mask=np.array(x.ie_mask, np.uint32))


def staged_flat_chain(kw, stages, stage_keys):
    """The chain in the tables of blance_plan_chains_ex: the base interned over the universe with every stage's node
    names (each state's slot range as wide as any stage's constraint), each stage's node fields and membership mask,
    and each stage's options as an option dict.  Returns (base tables, chain, stage option dicts, the interned plan of
    each stage's options: its ids, layout and constraints)."""
    prev, assign = kw["prev_map"], kw["partitions_to_assign"]
    T = len(stages)
    scs = []
    for _, rm, add, nw in stages:
        sc = {"nodesToRemove": rm, "nodesToAdd": add}
        if nw != "inherit":
            sc["nodeWeights"] = nw
        scs.append(sc)
    scs += [dict(keys, nodesToRemove=[], nodesToAdd=None) for keys in stage_keys]
    scs.append({"nodesToRemove": [], "nodesToAdd": None})
    o = options_of(kw)
    intern = lambda i: api.intern_scenario(prev, prev if assign is None else assign, kw["nodes_all"], kw["model"], o, scs, i)  # noqa: E731
    ip0 = intern(2 * T)
    base = C.tables_from_struct(abi.PlanIn.from_address(ip0.in_ptr))
    ips = [intern(T + t) for t in range(T)]
    opts = [option_dict(C.tables_from_struct(abi.PlanIn.from_address(ip.in_ptr)), base) for ip in ips]
    names = ip0.node_names
    N, NU = base.n_nodes, base.n_node_ids
    chain = []
    for nodes_all, rm, add, nw in stages:
        w = kw.get("node_weights") if nw == "inherit" else nw
        chain.append(dict(node_removed=np.array([names[q] in (rm or []) for q in range(NU)], np.uint8),
                          node_added=np.array([names[q] in (add or []) for q in range(NU)], np.uint8),
                          add_is_nil=int(add is None), has_node_weights=int(w is not None),
                          node_weight=np.array([(w or {}).get(names[q], 0) for q in range(N)], np.int32),
                          node_has_weight=np.array([names[q] in (w or {}) for q in range(N)], np.uint8),
                          node_in_all=np.array([names[q] in nodes_all for q in range(N)], np.uint8)))
    return base, chain, opts, ips
