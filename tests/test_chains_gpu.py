"""Chains of cluster changes on the device (blance_plan_chains): every stage of every chain equals the chain reference
of chain_util.py (the CPU oracle on one renumbered instance per stage), the net summary equals
blance_calc_partition_moves from the base's map to the last stage's, and nothing depends on the wave size, the engine
or the number of devices.  Needs an H100; run with `-m gpu`."""
import copy
import ctypes

import numpy as np
import pytest

import chain_util as C
from randgen import random_instance
from test_chains import flat_chain, literal_chain, make_chain
from test_scenarios import options_of, removal_allowed
from test_scenarios_gpu import random_base

import blance_b200
from blance_b200 import abi, synth, tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def random_chains(t, rng, n, T):
    """n chains of T stages over flat tables t: removals (the node leaves nodesAll at the next stage), re-additions,
    a removed id outside nodesAll, a node outside every stage's nodesAll, NodeWeights, nodesToAdd nil."""
    N, NU = t.n_nodes, t.n_node_ids
    k = int(np.maximum(t.state_constraints, 0).sum())
    chains = []
    for _ in range(n):
        members = np.ones(N, bool)
        if rng.random() < 0.3:
            members[int(rng.integers(N))] = False
        chain = []
        for s in range(T):
            rm, ad = np.zeros(NU, np.uint8), np.zeros(NU, np.uint8)
            inall = members.copy()
            r = rng.random()
            if r < 0.4 and members.sum() > k + 1:
                j = int(rng.choice(np.flatnonzero(members)))
                rm[j] = 1
                members[j] = False
            elif r < 0.7 and (~members).any():
                j = int(rng.choice(np.flatnonzero(~members)))
                members[j] = inall[j] = True
                ad[j] = 1
            elif r < 0.8 and NU > N:
                rm[N] = 1
            hw = int(rng.random() < 0.4)
            chain.append(dict(node_removed=rm, node_added=ad, add_is_nil=int(rng.random() < 0.15), has_node_weights=hw,
                              node_weight=rng.integers(-2, 7, N).astype(np.int32),
                              node_has_weight=(rng.random(N) < 0.8).astype(np.uint8), node_in_all=inall.astype(np.uint8)))
        if not t.part_in_prev.all():                 # plan.go:544: no removal in stage 1 with partitions absent from prevMap
            chain[0]["node_removed"][:] = 0
        chains.append(chain)
    return chains


def check_chains(ctx, base, chains, favor, opts=None, **kw):
    T = len(chains[0])
    res, nets = ctx.plan_chains(base, chains, favor, want_rows=[(i, t) for i in range(len(chains)) for t in range(T)],
                                opts=opts, **kw)
    for i, chain in enumerate(chains):
        ref, net = C.chain_reference(base, chain, None if opts is None else opts[i], favor)
        for t in range(T):
            C.assert_stage(res[i][t], ref[t], (i, t))
        assert np.array_equal(nets[i].node_ops, net["node_ops"]), i
        assert (nets[i].ops_total, nets[i].parts_moved) == (net["ops_total"], net["parts_moved"]), i
    return res, nets


@pytest.mark.parametrize("chunk", range(4))
def test_random_chains_match_chain_reference(ctx, chunk):
    for seed in range(chunk * 6, (chunk + 1) * 6):
        t, rng = random_base(seed)
        if t.part_in_assign.all() and rng.random() < 0.5:
            t.part_in_prev[:int(t.n_parts // 10)] = 0
            t.prev_rows[:int(t.n_parts // 10)] = -1
            t.prev_shape[:int(t.n_parts // 10)] = 0
        T = 1 + seed % 4
        check_chains(ctx, t, random_chains(t, rng, int(rng.integers(1, 6)), T), bool(seed % 2))


@pytest.mark.parametrize("chunk", range(3))
def test_string_instances_with_hierarchies_match_chain_reference(ctx, chunk):
    """Hierarchy rules, non-model prevMap states, names outside nodesAll: random string instances, one chain per call."""
    for seed in range(chunk * 30, (chunk + 1) * 30):
        kw = random_instance(seed)
        if not removal_allowed(kw) and kw["nodes_to_remove"]:
            continue
        stages = make_chain(kw, seed)
        if not removal_allowed(kw):
            stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
        base, chain, _ = flat_chain(kw, stages)
        if base.n_parts == 0:
            continue
        check_chains(ctx, base, [chain], bool(seed % 2))


def test_net_equals_calc_partition_moves(ctx):
    t, rng = random_base(11)
    chains = random_chains(t, rng, 3, 3)
    res, nets = check_chains(ctx, t, chains, False)
    a = t.part_in_assign != 0
    beg = np.where((t.part_in_prev != 0)[:, None], t.prev_rows, -1)[a]
    for i in range(3):
        end = res[i][2].next_rows[a]
        op_node, _, op_kind, op_count = ctx.calc_partition_moves(t.state_slot_off, beg, end, False)
        valid = np.arange(op_node.shape[1])[None, :] < op_count[:, None]
        ops = np.zeros((t.n_node_ids, 4), np.int64)
        np.add.at(ops, (op_node[valid], op_kind[valid]), 1)
        assert np.array_equal(ops, nets[i].node_ops)
        assert nets[i].ops_total == int(op_count.sum()) and nets[i].parts_moved == int((op_count > 0).sum())


def test_one_stage_equals_scenarios_ex(ctx):
    t, rng = random_base(4)
    t.state_has_stickiness[:] = 1
    chains = random_chains(t, rng, 5, 1)
    for ch in chains:
        ch[0]["node_in_all"][:] = 1
    opts = [{} if i % 2 else {"state_stickiness": np.full(t.n_states, i, np.int32)} for i in range(5)]
    res, _ = ctx.plan_chains(t, chains, True, want_rows=[(i, 0) for i in range(5)], opts=opts)
    scs = [{k: v for k, v in ch[0].items() if k != "node_in_all"} for ch in chains]
    sc = ctx.plan_scenarios(t, scs, True, want_rows=range(5), opts=opts)
    for i in range(5):
        for f in C.STAGE_FIELDS:
            assert np.array_equal(getattr(res[i][0], f), getattr(sc[i], f)), (i, f)
        for f in C.STAGE_SCALARS + ("sticky_steps",):
            assert getattr(res[i][0], f) == getattr(sc[i], f), (i, f)


def _same(a, b):
    for x, y in zip(a[0], b[0]):
        for u, v in zip(x, y):
            for f in C.STAGE_FIELDS:
                assert np.array_equal(getattr(u, f), getattr(v, f)), f
            for f in C.STAGE_SCALARS:
                assert getattr(u, f) == getattr(v, f), f
    for u, v in zip(a[1], b[1]):
        assert np.array_equal(u.node_ops, v.node_ops) and (u.ops_total, u.parts_moved) == (v.ops_total, v.parts_moved)


def test_results_do_not_depend_on_wave_engine_or_devices(ctx):
    t, rng = random_base(7)
    chains = random_chains(t, rng, 5, 3)
    want = [(i, s) for i in range(5) for s in range(3)]
    first = ctx.plan_chains(t, chains, False, want_rows=want)
    for mc in (1, 2, 0):
        _same(first, ctx.plan_chains(t, chains, False, max_concurrent=mc, want_rows=want))
    for engine in (1, 2):
        t.engine = engine
        _same(first, ctx.plan_chains(t, chains, False, want_rows=want))
    t.engine = 0
    import torch
    multi = tables.Context(device_ids=list(range(torch.cuda.device_count())))
    try:
        _same(first, multi.plan_chains(t, chains, False, want_rows=want))
    finally:
        multi.close()


def rolling_upgrade(t, nodes):
    """One chain per node j: take j out (nodesToRemove), then put it back (nodesAll again, nodesToAdd)."""
    N, NU = t.n_nodes, t.n_node_ids
    chains = []
    for j in nodes:
        rm, ad = np.zeros(NU, np.uint8), np.zeros(NU, np.uint8)
        rm[j] = ad[j] = 1
        out_j = np.ones(N, np.uint8)
        out_j[j] = 0
        zero = np.zeros(NU, np.uint8)
        chains.append([dict(node_removed=rm, node_added=zero, add_is_nil=0, node_in_all=np.ones(N, np.uint8)),
                       dict(node_removed=zero, node_added=ad, add_is_nil=0, node_in_all=np.ones(N, np.uint8))])
    return chains


def test_cfg4_reduced_rolling_upgrade(ctx):
    t = synth.make_rebalance(4, P=16384)
    chains = rolling_upgrade(t, range(8))
    res, _ = check_chains(ctx, t, chains, False)
    assert all(r[0].sticky_steps > 0 and r[1].sticky_steps > 0 for r in res)   # the speculative kernel ran on advanced state


def test_no_change_chain_equals_repeated_plans(ctx):
    """Repeated rebalances of a non-converging instance: stage t equals blance_plan_next_map on the tables the chain rule
    gives, advanced on the host from the previous call's rows."""
    t, rng = random_base(2)
    t.max_iters = 1
    NU, N = t.n_node_ids, t.n_nodes
    rm = np.zeros(NU, np.uint8)
    rm[0] = 1
    stage0 = dict(node_removed=rm, node_added=np.zeros(NU, np.uint8), add_is_nil=0, node_in_all=np.ones(N, np.uint8))
    rest = dict(node_removed=np.zeros(NU, np.uint8), node_added=np.zeros(NU, np.uint8), add_is_nil=0,
                node_in_all=np.r_[0, np.ones(N - 1)].astype(np.uint8))
    chain = [stage0, rest, rest]
    res, _ = ctx.plan_chains(t, [chain], False, want_rows=[(0, s) for s in range(3)])
    cur = t
    for s in range(3):
        x = C.substituted(cur, chain[s], None, s)
        y, order = C.renumbered(x, chain[s]["node_in_all"])
        r = ctx.plan_next_map(y)
        nxt = np.where(r.next_rows >= 0, order[np.maximum(r.next_rows, 0)], -1).astype(np.int32)
        assert np.array_equal(res[0][s].next_rows, nxt), s
        assert (res[0][s].iters_run, res[0][s].converged, res[0][s].steps) == (r.iters_run, r.converged, r.steps), s
        cur = C.advance(cur, nxt, r.next_shape)
    assert not res[0][0].converged


def test_node_removed_any_nonzero_means_removed(ctx):
    t, _ = random_base(9)
    t.node_removed[:] = 0
    t.node_removed[[0, 2]] = 1
    one = ctx.plan_next_map(t)
    # 2 and 6 leave bit 0 (NR_REMOVE) clear: only the normalisation makes them "removed"
    for v in (7, 2, 6):
        t2 = copy.copy(t)
        t2.node_removed = np.where(t.node_removed != 0, v, 0).astype(np.uint8)
        other = ctx.plan_next_map(t2)
        assert np.array_equal(one.next_rows, other.next_rows) and np.array_equal(one.warn, other.warn), v
        assert (one.iters_run, one.converged, one.steps) == (other.iters_run, other.converged, other.steps), v


def test_errors_leave_the_context_usable(ctx):
    t, rng = random_base(3)
    chains = random_chains(t, rng, 2, 2)
    bad = copy.deepcopy(chains)
    bad[1][1]["node_in_all"] = bad[1][1]["node_in_all"] * 3
    with pytest.raises(blance_b200.BlanceError, match="chain 1, stage 1: node_in_all"):
        ctx.plan_chains(t, bad, False)
    lib = ctx.lib
    base = t.struct()
    assert lib.blance_plan_chains(ctx.ptr, ctypes.byref(base), 0, 1, (abi.ChainStage * 1)(), None, 0, 0,
                                  (abi.ScenarioOut * 1)(), None) == -1
    check_chains(ctx, t, chains, False)


# ---- the string API (PlanNextMapChains) --------------------------------------------------------------------------

def _string_chains(stages, explicit):
    out = []
    for nodes_all, rm, add, nw in stages:
        st = {"nodesToRemove": rm, "nodesToAdd": add}
        if nw != "inherit":
            st["nodeWeights"] = nw
        if explicit:
            st["nodesAll"] = nodes_all
        out.append(st)
    return [{"stages": out}]


@pytest.mark.parametrize("chunk", range(2))
def test_string_api_matches_literal_loop(chunk):
    """PlanNextMapChains on string maps against the literal oracle driven as the Go loop; the default nodesAll rule
    where the stages leave it out; the caller's maps are not mutated."""
    for seed in range(chunk * 40, (chunk + 1) * 40):
        kw = random_instance(seed)
        if not removal_allowed(kw) and kw["nodes_to_remove"]:
            continue
        stages = make_chain(kw, seed)
        if not removal_allowed(kw):
            stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
        lit = literal_chain(kw, stages)
        prev = kw["prev_map"]
        assign = prev if kw["partitions_to_assign"] is None else kw["partitions_to_assign"]
        before = (copy.deepcopy(prev), copy.deepcopy(assign))
        # the stages' own nodesAll when one node stays outside all of them, else the default rule
        explicit = len(stages[0][0]) != len(kw["nodes_all"]) or seed % 3 == 0
        res = blance_b200.PlanNextMapChains(prev, assign, kw["nodes_all"], kw["model"], options_of(kw),
                                            _string_chains(stages, explicit), favorMinNodes=bool(seed % 2), wantMaps=[0])
        for t, (l, r) in enumerate(zip(lit, res[0]["stages"])):
            want = l["next_map"] if r["iterations"] > 0 else {}
            assert r["next_map"] == want, (seed, t)
            assert r["warnings"] == (l["warnings"] if r["iterations"] > 0 else {}), (seed, t)
            assert r["iterations"] == l["iterations"], (seed, t)
        assert (prev, assign) == before, seed


def test_string_api_no_change_chain_equals_repeated_plan_next_map_ex():
    """Repeated rebalances of an instance that does not converge in one iteration: each stage equals PlanNextMapEx
    through the string API on the maps the previous call left, with the per-node ops of each stage summed and net."""
    for seed in range(400):
        kw = random_instance(seed)
        holds = any(kw["nodes_all"][0] in (nodes or []) for nbs in kw["prev_map"].values() for nodes in nbs.values())
        if kw["partitions_to_assign"] is None and len(kw["prev_map"]) > 8 and len(kw["nodes_all"]) > 4 and holds:
            break
    kw["nodes_to_remove"], kw["nodes_to_add"] = [kw["nodes_all"][0]], []
    o = options_of(kw)
    o.MaxIterationsPerPlan = 1
    stages = [{"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": []}] + [{"nodesToRemove": [], "nodesToAdd": []}] * 2
    prev = copy.deepcopy(kw["prev_map"])
    res = blance_b200.PlanNextMapChains(prev, prev, kw["nodes_all"], kw["model"], o, [{"stages": stages}], wantMaps=[0])
    cur = copy.deepcopy(kw["prev_map"])
    nodes = list(kw["nodes_all"])
    for t, st in enumerate(stages):
        p, a = copy.deepcopy(cur), copy.deepcopy(cur)
        nxt, warnings = blance_b200.PlanNextMapEx(p, a, nodes, st["nodesToRemove"], st["nodesToAdd"], kw["model"], o)
        got = res[0]["stages"][t]
        assert got["next_map"] == nxt and got["warnings"] == warnings, t
        cur = dict(cur)
        cur.update(copy.deepcopy(nxt))
        nodes = [n for n in nodes if n not in st["nodesToRemove"]]
    assert not all(s["converged"] for s in res[0]["stages"])
