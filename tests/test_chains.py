"""Chains of cluster changes (blance_plan_chains), CPU side: the chain reference of chain_util.py - one plain
renumbered instance per stage, planned by the fast oracle - against the literal oracle driven as the Go host loop on
string maps, argument checks without a device, and the ABI.  The device path is tests/test_chains_gpu.py."""
import copy
import ctypes
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import chain_util as C
import golden_util as G
from oracle_loader import literal
from randgen import random_instance
from test_scenarios import OUTSIDE, options_of, removal_allowed

import blance_b200
from blance_b200 import _host, abi, api, tables

L = literal()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_chain(kw, seed):
    """2-3 stages over kw's universe (nodes_all): the case's own node sets first, then node removals, re-additions
    (the node keeps its position), a removed name outside nodesAll, NodeWeights changes and no-change rebalances.
    Sometimes one node stays outside every stage's nodesAll.  A stage is (nodesAll_t, remove, add, nodeWeights or
    "inherit")."""
    rnd = random.Random(seed * 31 + 7)
    universe = kw["nodes_all"]
    never = universe[-1] if len(universe) > 2 and rnd.random() < 0.2 else None
    in_order = lambda names: [n for n in universe if n in names and n != never]
    rm0 = kw["nodes_to_remove"]
    stages = [(in_order(set(universe)), rm0, kw["nodes_to_add"], "inherit")]
    members = set(in_order(set(universe))) - set(rm0 or [])
    for _ in range(rnd.randint(1, 2)):
        r = rnd.random()
        absent = [n for n in universe if n not in members and n != never]
        nw = "inherit" if rnd.random() < 0.6 else rnd.choice([None, {n: rnd.randint(-2, 4) for n in universe if rnd.random() < 0.7}])
        if r < 0.35 and members:
            j = rnd.choice(sorted(members))
            stages.append((in_order(members), [j], [], nw))
            members = members - {j}
        elif r < 0.6 and absent:
            j = rnd.choice(absent)
            members = members | {j}
            stages.append((in_order(members), [], [j], nw))
        elif r < 0.75:
            stages.append((in_order(members), [OUTSIDE], None, nw))
        else:
            stages.append((in_order(members), [], rnd.choice([[], None]), nw))
    return stages


def literal_chain(kw, stages):
    """The Go host loop of include/blance_b200.h on string maps with the literal oracle."""
    prev = copy.deepcopy(kw["prev_map"])
    assign = copy.deepcopy(kw["partitions_to_assign"])
    out = []
    for nodes_all, rm, add, nw in stages:
        k = copy.deepcopy(kw)
        k.update(prev_map=copy.deepcopy(prev), partitions_to_assign=copy.deepcopy(assign), nodes_all=list(nodes_all),
                 nodes_to_remove=copy.deepcopy(rm), nodes_to_add=copy.deepcopy(add))
        if nw != "inherit":
            k["node_weights"] = copy.deepcopy(nw)
        lit = L.plan_next_map_ex(**k)
        out.append(lit)
        nxt = lit["next_map"]
        prev = dict(prev)
        prev.update(copy.deepcopy(nxt))
        assign = copy.deepcopy(nxt)
    return out


def flat_chain(kw, stages):
    """The chain in the tables of blance_plan_chains: the base interned over the universe with every stage's node
    names, and each stage's node fields and membership mask in those ids.  Returns (base tables, chain, interned)."""
    prev, assign = kw["prev_map"], kw["partitions_to_assign"]
    scs = []
    for _, rm, add, nw in stages:
        sc = {"nodesToRemove": rm, "nodesToAdd": add}
        if nw != "inherit":
            sc["nodeWeights"] = nw
        scs.append(sc)
    ip = api.intern_scenario(prev, prev if assign is None else assign, kw["nodes_all"], kw["model"], options_of(kw), scs, 0)
    names = ip.node_names
    base = C.tables_from_struct(abi.PlanIn.from_address(ip.in_ptr))
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
    return base, chain, ip


def unintern(ip, t, stage):
    """(next_map, warnings) of one stage of the chain reference, through the host layer's own uninterning."""
    out = _host.plan_out(ip)
    po = abi.PlanOut.from_address(out.out_ptr)
    rows = np.ascontiguousarray(stage["next_rows"], np.int32)
    if rows.size:
        ctypes.memmove(po.next_rows, rows.ctypes.data, rows.nbytes)
    for f in ("next_shape", "warn"):
        a = np.ascontiguousarray(stage[f], np.uint8)
        if a.size:
            ctypes.memmove(getattr(po, f), a.ctypes.data, a.nbytes)
    po.iters_run, po.converged, po.steps = stage["iters_run"], stage["converged"], stage["steps"]
    if po.iters_run <= 0:
        return {}, {}
    return _host.unintern_plan(ip, out)


def check_chain(kw, seed):
    if not removal_allowed(kw) and kw["nodes_to_remove"]:
        return
    stages = make_chain(kw, seed)
    if not removal_allowed(kw):       # plan.go:544 panics on a removal in stage 1 only: later stages have every partition
        stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
    lit = literal_chain(kw, stages)
    base, chain, ip = flat_chain(kw, stages)
    ref, net = C.chain_reference(base, chain, None, bool(seed % 2))
    for t, (l, r) in enumerate(zip(lit, ref)):
        next_map, warnings = unintern(ip, t, r)
        assert next_map == l["next_map"], (seed, t)
        assert warnings == l["warnings"], (seed, t)
        assert r["iters_run"] == l["iterations"], (seed, t)
    assert net["ops_total"] == int(net["node_ops"].sum())
    assert net["parts_moved"] <= base.n_parts


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_chain_reference_matches_literal_loop_golden(c):
    check_chain(G.plan_kwargs(c), c["index"])


@pytest.mark.parametrize("chunk", range(6))
def test_chain_reference_matches_literal_loop_random(chunk):
    for seed in range(chunk * 40, (chunk + 1) * 40):
        check_chain(random_instance(seed), seed)


def test_a_partition_to_assign_with_a_non_model_state_is_rejected():
    """Stage 2's extra_tot_first is stage 1's extra_tot_rest because a next row holds model states only: the host
    layer rejects a partitionsToAssign entry with another state (the reference panics on it, plan.go:148)."""
    prev = {"0": {"primary": ["a"], "dead": ["b"]}}
    assign = {"0": {"primary": ["a"], "dead": ["b"]}}
    with pytest.raises(Exception, match="not in the model"):
        api.intern_scenario(prev, assign, ["a", "b"], {"primary": (0, 1)}, None,
                            [{"nodesToRemove": [], "nodesToAdd": None}], 0)


def test_renumbering_keeps_a_full_membership_unchanged():
    kw = random_instance(5)
    base, chain, _ = flat_chain(kw, make_chain(kw, 5))
    x = C.substituted(base, chain[0], None, 0)
    r, order = C.renumbered(x, np.ones(base.n_nodes, np.uint8))
    assert np.array_equal(order, np.arange(base.n_node_ids))
    assert np.array_equal(r.prev_rows, x.prev_rows) and np.array_equal(r.ie_mask, x.ie_mask)


# ---- argument checks without a device ---------------------------------------------------------------------------

def _chain_args(t, chains):
    T = len(chains[0])
    keep, sts = [], (abi.ChainStage * (len(chains) * T))()
    for i, ch in enumerate(chains):
        for k, stage in enumerate(ch):
            s = sts[i * T + k]
            for f in tables.SCENARIO_FIELDS:
                v = stage.get(f, getattr(t, f))
                if f in ("add_is_nil", "has_node_weights"):
                    setattr(s.nodes, f, int(v))
                    continue
                a = np.ascontiguousarray(v, np.int32 if f == "node_weight" else np.uint8)
                keep.append(a)
                setattr(s.nodes, f, a.ctypes.data)
            m = stage.get("node_in_all", np.ones(t.n_nodes, np.uint8))
            if m is None:
                s.node_in_all = None
            else:
                a = np.ascontiguousarray(m, np.uint8)
                keep.append(a)
                s.node_in_all = a.ctypes.data
    outs = (abi.ScenarioOut * (len(chains) * T))()
    return keep, sts, outs


def _null_ctx_call(t, chains, n_stages=None):
    lib = abi.capi()
    keep, sts, outs = _chain_args(t, chains)
    base = t.struct()
    st = lib.blance_plan_chains(None, ctypes.byref(base), len(chains), len(chains[0]) if n_stages is None else n_stages, sts,
                                None, 0, 0, outs, None)
    return st, lib.blance_last_error(None).decode()


def _small():
    t = tables.PlanTables(4, 2, 6, [0, 1], [1, 1])
    t.part_in_prev[:] = 1
    return t


def test_argument_errors_name_chain_and_stage():
    t = _small()
    ok = {}
    st, msg = _null_ctx_call(t, [[ok, ok], [ok, {"add_is_nil": 2}]])
    assert st == -1 and "chain 1, stage 1: add_is_nil" in msg
    st, msg = _null_ctx_call(t, [[ok, {"node_in_all": np.array([1, 2, 1, 1])}]])
    assert st == -1 and "chain 0, stage 1: node_in_all is neither 0 nor 1" in msg
    st, msg = _null_ctx_call(t, [[{"node_in_all": None}]])
    assert st == -1 and "chain 0, stage 0: node_in_all is NULL" in msg
    st, msg = _null_ctx_call(t, [[ok]], n_stages=0)
    assert st == -1 and "n_stages must be positive" in msg
    t.max_iters = 0
    st, msg = _null_ctx_call(t, [[ok, ok]])
    assert st == -1 and "max_iters >= 1" in msg
    t.max_iters = 10
    st, msg = _null_ctx_call(t, [[ok, ok]])
    assert st == -1 and msg == "ctx is NULL"


def test_chain_struct_layout_matches_header():
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu\n", sizeof(blance_chain_stage), offsetof(blance_chain_stage, node_in_all),
             sizeof(blance_chain_out), offsetof(blance_chain_out, ops_total), offsetof(blance_chain_out, parts_moved));
      return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")], check=True)
        out = list(map(int, subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    S, O = abi.ChainStage, abi.ChainOut
    assert out == [ctypes.sizeof(S), S.node_in_all.offset, ctypes.sizeof(O), O.ops_total.offset, O.parts_moved.offset]


def _have_gpu():
    lib = abi.capi()
    ctx = ctypes.c_void_p()
    st = lib.blance_ctx_create(ctypes.byref(ctx), -1)
    if st == 0:
        lib.blance_ctx_destroy(ctx)
    return st == 0


def test_no_cpu_fallback_for_chains():
    if _have_gpu():
        pytest.skip("a CUDA device is present")
    with pytest.raises(blance_b200.BlanceError):
        tables.Context().plan_chains(_small(), [[{}, {}]], False)


# ---- the string API (PlanNextMapChains): checks before any device work --------------------------------------------

def _string_chain(stages):
    return [{"stages": [{"nodesToRemove": rm, "nodesToAdd": ad} for rm, ad in stages]}]


def test_string_api_rejects_before_device_work():
    prev = {"0": {"primary": ["a"]}}
    assign = {"0": {"primary": ["a"]}, "1": {}}          # "1" is missing from prevMap
    model = {"primary": (0, 1)}
    # a removal in stage 1 with an assigned partition absent from prevMap: the reference panics (plan.go:544)
    with pytest.raises(blance_b200.BlanceError, match="chain 0, stage 0: "):
        blance_b200.PlanNextMapChains(prev, assign, ["a", "b"], model, None, _string_chain([(["a"], None), ([], None)]))
    # chains of different lengths
    chains = _string_chain([([], None)]) + _string_chain([([], None), ([], None)])
    with pytest.raises(blance_b200.BlanceError, match="chain 1 has 2 stages"):
        blance_b200.PlanNextMapChains(prev, prev, ["a", "b"], model, None, chains)
    # a stage's nodesAll names a node outside the universe
    chains = [{"stages": [{"nodesToRemove": [], "nodesToAdd": None, "nodesAll": ["a", "zz"]}]}]
    with pytest.raises(blance_b200.BlanceError, match="chain 0, stage 0: NodesAll name 'zz'"):
        blance_b200.PlanNextMapChains(prev, prev, ["a", "b"], model, None, chains)
    with pytest.raises(ValueError, match="chain 0, stage 1 lacks nodesToAdd"):
        blance_b200.PlanNextMapChains(prev, prev, ["a", "b"], model, None,
                                      [{"stages": [{"nodesToRemove": [], "nodesToAdd": []}, {"nodesToRemove": []}]}])


def test_no_cpu_fallback_for_string_chains():
    if _have_gpu():
        pytest.skip("a CUDA device is present")
    with pytest.raises(blance_b200.BlanceError):
        blance_b200.PlanNextMapChains({}, {"0": {}}, ["a"], {"primary": (0, 1)}, None, _string_chain([([], ["a"])]))
