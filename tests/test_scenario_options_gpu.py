"""What-if scenarios that vary plan options on the device (blance_plan_scenarios_ex): every scenario's plan equals
the CPU oracle on its substituted tables, every summary equals a host recomputation with the scenario's own
partition weights, and nothing depends on the wave size, the engine or the number of devices.  Needs an H100; run
with `-m gpu`."""
import copy
import ctypes

import numpy as np
import pytest

import golden_util as G
from oracle_loader import fast_lib_path

import blance_b200
from blance_b200 import abi, synth, tables

pytestmark = pytest.mark.gpu

FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
FAST.oracle_fast_calc_partition_moves.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 4


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def oracle_tables(t):
    r = tables.PlanResult(t)
    s = t.struct()
    assert FAST.oracle_fast_plan_next_map(ctypes.byref(s), ctypes.byref(r.out)) == 0
    return r


def reference_summary(t, next_rows, warn, favor_min_nodes):
    """The summaries of blance_plan_scenarios recomputed on the host (as tests/test_scenarios_gpu.py does):
    CalcPartitionMoves (fast oracle) from the pristine prev row to the next row of every assigned partition, and
    countStateNodes over the final map weighted with t's partition weights."""
    assigned = t.part_in_assign != 0
    in_prev = t.part_in_prev != 0
    NU, S, SL = t.n_node_ids, t.n_states, t.n_slots
    beg = np.ascontiguousarray(np.where(in_prev[:, None], t.prev_rows, -1).astype(np.int32)[assigned])
    end = np.ascontiguousarray(next_rows[assigned], np.int32)
    n = int(assigned.sum())
    max_ops = max(1, 2 * SL)
    op_node = np.zeros((max(n, 1), max_ops), np.int32)
    op_state = np.zeros((max(n, 1), max_ops), np.uint8)
    op_kind = np.zeros((max(n, 1), max_ops), np.uint8)
    op_count = np.zeros(max(n, 1), np.int32)
    slot_off = np.ascontiguousarray(t.state_slot_off, np.int32)
    if n:
        assert FAST.oracle_fast_calc_partition_moves(n, S, S, slot_off.ctypes.data, beg.ctypes.data, end.ctypes.data,
                                                     int(favor_min_nodes), max_ops, op_node.ctypes.data, op_state.ctypes.data,
                                                     op_kind.ctypes.data, op_count.ctypes.data) == 0
    node_ops = np.zeros((NU, 4), np.int64)
    valid = np.arange(max_ops)[None, :] < op_count[:n, None]
    np.add.at(node_ops, (op_node[:n][valid], op_kind[:n][valid]), 1)
    final = np.where(assigned[:, None], next_rows, t.prev_rows)
    include = assigned | in_prev
    w = np.where((t.has_part_weights != 0) & (t.part_has_weight != 0), t.part_weight, 1).astype(np.int64)
    load = np.zeros((S, NU), np.int64)
    for s in range(S):
        blk = final[include, t.state_slot_off[s]:t.state_slot_off[s + 1]]
        ww = np.broadcast_to(w[include][:, None], blk.shape)
        ok = blk >= 0
        np.add.at(load[s], blk[ok], ww[ok])
    return dict(node_ops=node_ops, state_node_load=load, parts_moved=int((op_count[:n] > 0).sum()),
                ops_total=int(op_count[:n].sum()), warn_parts=int(warn[assigned].any(axis=1).sum()))


def assert_scenario(got, ref, summ, what):
    assert np.array_equal(got.next_rows, ref.next_rows), what
    assert np.array_equal(got.next_shape, ref.next_shape) and np.array_equal(got.warn, ref.warn), what
    assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps), what
    assert np.array_equal(got.node_ops, summ["node_ops"]), what
    assert np.array_equal(got.state_node_load, summ["state_node_load"]), what
    assert (got.parts_moved, got.ops_total, got.warn_parts) == (summ["parts_moved"], summ["ops_total"], summ["warn_parts"]), what


def check_against_oracle(ctx, base, scs, opts, favor, **kw):
    res = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), opts=opts, **kw)
    for i, (sc, o, got) in enumerate(zip(scs, opts, res)):
        t = tables.scenario_tables(base, sc, o)
        ref = oracle_tables(t)
        assert_scenario(got, ref, reference_summary(t, ref.next_rows, ref.warn, favor), i)
    return res


def rack_masks(t, rack, states_with_rule):
    """A different-rack rule (racks of `rack` consecutive nodes) on the given states: rule_off, ie_mask, n_rules.
    Anchors outside nodesAll and "" allow every node."""
    N, NU, S = t.n_nodes, t.n_node_ids, t.n_states
    HW = (N + 31) // 32
    rule_off = np.zeros(S + 1, np.int32)
    for s in range(S):
        rule_off[s + 1] = rule_off[s] + (1 if s in states_with_rule else 0)
    R = int(rule_off[-1])
    bits = np.zeros((NU + 1, N), bool)
    for a in range(NU + 1):
        bits[a] = True
        if a < N:
            bits[a, (a // rack) * rack:(a // rack + 1) * rack] = False
    words = np.zeros((NU + 1, HW), np.uint32)
    for q in range(N):
        words[:, q >> 5] |= (bits[:, q].astype(np.uint32) << np.uint32(q & 31))
    return rule_off, np.ascontiguousarray(np.broadcast_to(words, (R, NU + 1, HW)).reshape(-1)), R


def random_base(seed):
    """Mid-size random flat instances (as tests/test_scenarios_gpu.py draws them), with every state's slot range one
    wider than its constraints so that scenarios can raise them."""
    rng = np.random.default_rng(seed + 2000)
    N = int(rng.integers(8, 160))
    S = int(rng.integers(1, 4))
    k = [int(rng.integers(1, 4)) if s < 2 else int(rng.integers(0, 2)) for s in range(S)]
    if np.random.default_rng([seed, 4]).random() < 0.25:   # k = 4 from a stream of its own: other seeds keep their instances
        k[0] = 4
    while sum(k) + S > N - 2:
        k = [max(1, x - 1) if s == 0 else max(0, x - 1) for s, x in enumerate(k)]
    P = int(rng.integers(70, 2500))
    NU = N + int(rng.integers(0, 3))
    t = tables.PlanTables(N, S, P, list(range(S)), k, n_node_ids=NU)
    SL = t.n_slots
    rows = np.full((P, SL), -1, np.int32)
    live = max(SL + 1, N - int(rng.integers(0, 4)))
    for p in range(P):
        perm = rng.permutation(live)[:SL]
        for s in range(S):
            lo, hi = int(t.state_slot_off[s]), int(t.state_slot_off[s + 1])
            n = hi - lo if rng.random() < 0.9 else int(rng.integers(0, hi - lo + 1))
            rows[p, lo:lo + n] = perm[lo:lo + n]
    if NU > N and P > 3:
        rows[1, SL - 1] = N
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:] = 2
    t.cur_shape[:] = 2
    t.part_in_prev[:] = 1
    if rng.random() < 0.3:
        t.part_in_assign[:] = (rng.random(P) < 0.8).astype(np.uint8)
    if rng.random() < 0.6:
        t.has_part_weights = 1
        t.part_has_weight[:] = (rng.random(P) < 0.4).astype(np.uint8)
        t.part_weight[:] = rng.integers(1, 9, P)
        t.state_has_stickiness[:] = (rng.random(S) < 0.7).astype(np.uint8)
        t.state_stickiness[:] = rng.integers(0, 5, S)
    if rng.random() < 0.4 and S > 1:
        t.has_hier_rules = 1
        t.rule_off, t.ie_mask, t.n_rules = rack_masks(t, 4, {1})
    t.booster_kind = int(rng.random() < 0.3)
    t.max_iters = int(rng.integers(1, 6))
    return tables.widen_layout(t, np.asarray(k) + 1), rng


def random_option(t, rng):
    """One scenario's option dict: any subset of the four groups, with random values within the limits."""
    S, P = t.n_states, t.n_parts
    o = {}
    if rng.random() < 0.5:
        width = np.diff(t.state_slot_off)
        o["state_constraints"] = np.array([int(rng.integers(max(0, int(t.state_constraints[s]) - 1), min(4, int(width[s])) + 1))
                                           for s in range(S)], np.int32)
        o["state_constraints"][0] = max(1, o["state_constraints"][0])
    if rng.random() < 0.5:
        o["state_stickiness"] = rng.integers(0, 9, S).astype(np.int32)
        o["state_has_stickiness"] = (rng.random(S) < 0.7).astype(np.uint8)
    if rng.random() < 0.6:
        o["has_part_weights"] = int(rng.random() < 0.85)
        k = int(rng.integers(0, max(1, P // 20)))
        part = rng.permutation(P)[:k].astype(np.int32)
        o["weight_overrides"] = (part, rng.integers(-3, 40, k).astype(np.int32), (rng.random(k) < 0.8).astype(np.uint8))
    if rng.random() < 0.3 and S > 1:
        if t.has_hier_rules and rng.random() < 0.5:
            o["has_hier_rules"] = 0
        else:
            o["has_hier_rules"] = 1
            o["rule_off"], o["ie_mask"], o["n_rules"] = rack_masks(t, int(rng.integers(2, 9)), {1})
            o["n_hier_bits"] = t.n_nodes
    return o


def random_scenarios(t, rng, count):
    N, NU = t.n_nodes, t.n_node_ids
    scs, opts = [], []
    for i in range(count):
        rm = np.zeros(NU, np.uint8)
        if t.part_in_prev.all():
            rm[rng.permutation(NU)[:int(rng.integers(0, max(1, N // 8)))]] = 1
        ad = np.zeros(NU, np.uint8)
        ad[rng.permutation(N)[:int(rng.integers(0, N // 4 + 1))]] = 1
        scs.append(dict(node_removed=rm, node_added=ad, add_is_nil=int(rng.random() < 0.15), has_node_weights=0,
                        node_weight=np.zeros(N, np.int32), node_has_weight=np.zeros(N, np.uint8)))
        opts.append({} if i == 0 else random_option(t, rng))
    return scs, opts


@pytest.mark.parametrize("chunk", range(4))
def test_random_option_scenarios_match_oracle_and_reference_summary(ctx, chunk):
    for seed in range(chunk * 8, (chunk + 1) * 8):
        t, rng = random_base(seed)
        scs, opts = random_scenarios(t, rng, int(rng.integers(1, 12)))
        check_against_oracle(ctx, t, scs, opts, bool(seed % 2))


def _same_results(a, b):
    for x, y in zip(a, b):
        for f in ("next_rows", "next_shape", "warn", "node_ops", "state_node_load"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), f
        for f in ("iters_run", "converged", "steps", "parts_moved", "ops_total", "warn_parts"):
            assert getattr(x, f) == getattr(y, f), f


def test_no_opts_and_inherited_opts_equal_plan_scenarios(ctx):
    t, rng = random_base(11)
    scs, _ = random_scenarios(t, rng, 5)
    plain = ctx.plan_scenarios(t, scs, False, want_rows=range(5))
    _same_results(plain, ctx.plan_scenarios(t, scs, False, want_rows=range(5), opts=[{}] * 5))
    # a NULL opts array through the _ex entry point
    base = t.struct()
    results = [tables.ScenarioResult(t, True) for _ in scs]
    outs = (abi.ScenarioOut * 5)(*[r.out for r in results])
    arr = (abi.Scenario * 5)()
    arrays = []
    for i, sc in enumerate(scs):
        for f in tables.SCENARIO_FIELDS:
            v = sc[f]
            if f in ("add_is_nil", "has_node_weights"):
                setattr(arr[i], f, int(v))
            else:
                a = np.ascontiguousarray(v, dtype=np.int32 if f == "node_weight" else np.uint8)
                arrays.append(a)
                setattr(arr[i], f, a.ctypes.data)
    assert ctx.lib.blance_plan_scenarios_ex(ctx.ptr, ctypes.byref(base), 5, arr, None, 0, 0, outs) == 0
    for r, o in zip(results, outs):
        r.out = o
    _same_results(plain, results)


def test_results_do_not_depend_on_wave_engine_or_devices(ctx):
    t, rng = random_base(7)
    scs, opts = random_scenarios(t, rng, 7)
    first = ctx.plan_scenarios(t, scs, False, want_rows=range(7), opts=opts)
    for mc in (1, 3, 0):
        _same_results(first, ctx.plan_scenarios(t, scs, False, max_concurrent=mc, want_rows=range(7), opts=opts))
    for engine in (0, 1, 2):
        t.engine = engine
        res = ctx.plan_scenarios(t, scs, False, want_rows=range(7), opts=opts)
        for x, y in zip(first, res):              # sticky_steps counts what the engine did; everything else is equal
            for f in ("next_rows", "next_shape", "warn", "node_ops", "state_node_load"):
                assert np.array_equal(getattr(x, f), getattr(y, f)), f
            assert (x.iters_run, x.converged, x.steps, x.parts_moved, x.ops_total) == (y.iters_run, y.converged, y.steps, y.parts_moved, y.ops_total)
    t.engine = 0
    import torch
    multi = tables.Context(device_ids=list(range(torch.cuda.device_count())))
    try:
        _same_results(first, multi.plan_scenarios(t, scs, False, want_rows=range(7), opts=opts))
    finally:
        multi.close()


def test_lone_scenario_with_weight_overrides(ctx):
    """A device's only scenario is planned on the base upload itself; its weight overrides must still apply."""
    t, rng = random_base(5)
    t.has_part_weights = 1
    scs, _ = random_scenarios(t, rng, 1)
    part = np.arange(0, t.n_parts, 7, dtype=np.int32)
    o = dict(weight_overrides=(part, (part % 13 + 2).astype(np.int32), np.ones(len(part), np.uint8)))
    check_against_oracle(ctx, t, scs, [o], False)


def _fresh_then_rebalance(ctx, cfg, **size):
    fresh = synth.make_fresh(cfg, **size)
    rows = ctx.plan_next_map(fresh).next_rows
    return synth.make_rebalance(cfg, prev_rows=rows, **size)


def _same_nodes(t, n):
    return [dict(node_removed=t.node_removed.copy(), node_added=t.node_added.copy(), add_is_nil=int(t.add_is_nil))
            for _ in range(n)]


def test_cfg2_replicas_and_rack_rule(ctx):
    t = tables.widen_layout(_fresh_then_rebalance(ctx, 2), [1, 2])
    two = np.array([1, 2], np.int32)
    opts = [{}, dict(state_constraints=two), dict(has_hier_rules=0), dict(state_constraints=two, has_hier_rules=0)]
    check_against_oracle(ctx, t, _same_nodes(t, len(opts)), opts, False)


def test_cfg4_reduced_option_sweep(ctx):
    base = synth.make_rebalance(4, P=16384)
    t = tables.widen_layout(base, [1, 3])
    S = t.n_states
    opts = [dict(state_stickiness=np.full(S, v, np.int32), state_has_stickiness=np.ones(S, np.uint8)) for v in (0, 1, 2, 3, 5, 8)]
    opts.append(dict(state_constraints=np.array([1, 3], np.int32)))
    rng = np.random.default_rng(4)
    part = rng.permutation(t.n_parts)[:t.n_parts // 100].astype(np.int32)
    opts.append(dict(weight_overrides=(part, rng.integers(1, 50, len(part)).astype(np.int32), np.ones(len(part), np.uint8))))
    opts.append({})
    res = check_against_oracle(ctx, t, _same_nodes(t, len(opts)), opts, False)
    # the speculative kernel ran inside the wave where the base configuration makes it eligible
    assert res[-1].sticky_steps > 0 and res[-2].sticky_steps > 0


def test_constraints_of_4_plan_as_lockstep(ctx):
    t = tables.scenario_tables(tables.widen_layout(synth.make_rebalance(4, P=16384), [1, 4]), {},
                               dict(state_constraints=np.array([1, 4], np.int32)))
    auto = ctx.plan_next_map(t)
    t.engine = 1
    lock = ctx.plan_next_map(t)
    assert np.array_equal(auto.next_rows, lock.next_rows) and auto.iters_run == lock.iters_run


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_string_api_options_per_scenario(c):
    kw = G.plan_kwargs(c)
    prev = kw["prev_map"]
    assign = kw["partitions_to_assign"] if kw["partitions_to_assign"] is not None else prev
    before = (copy.deepcopy(prev), copy.deepcopy(assign))
    sc = {"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": kw["nodes_to_add"],
          "modelStateConstraints": kw["model_state_constraints"], "partitionWeights": kw["partition_weights"],
          "stateStickiness": kw["state_stickiness"], "nodeWeights": kw["node_weights"],
          "nodeHierarchy": kw["node_hierarchy"], "hierarchyRules": kw["hierarchy_rules"]}
    o = blance_b200.PlanNextMapOptions(NodeScoreBooster=kw["booster"])
    r = blance_b200.PlanNextMapScenarios(prev, assign, kw["nodes_all"], kw["model"], o, [sc, sc], wantMaps=[0, 1])
    for x in r:
        assert x["next_map"] == G.pmap(c["exp"])
        assert G.count_warnings(c, x["warnings"]) == c["expNumWarnings"]
    assert (prev, assign) == before                      # no side effects on the caller's maps


def test_errors_leave_the_context_usable(ctx):
    t, rng = random_base(3)
    scs, _ = random_scenarios(t, rng, 2)
    P = t.n_parts
    width = np.diff(t.state_slot_off)
    one = np.ones(1, np.uint8)
    cases = [
        (dict(has_part_weights=2), "has_part_weights is neither"),
        (dict(weight_overrides=(np.array([P], np.int32), np.ones(1, np.int32), one)), "outside \\[0, n_parts\\)"),
        (dict(weight_overrides=(np.array([1, 1], np.int32), np.ones(2, np.int32), np.ones(2, np.uint8))), "two weight overrides"),
        (dict(weight_overrides=(np.array([0], np.int32), np.array([1000000000], np.int32), one)), "above 999999999"),
        (dict(has_part_weights=1, weight_overrides=(np.array([0], np.int32), np.array([999999999], np.int32), one)), "exceeds int32"),
        (dict(weight_overrides=(np.array([0], np.int32), np.ones(1, np.int32), np.array([2], np.uint8))), "ow_has is neither"),
        (dict(state_constraints=(width + 1).astype(np.int32)), "slot range is smaller"),
        (dict(state_stickiness=np.zeros(t.n_states, np.int32), state_has_stickiness=np.full(t.n_states, 2, np.uint8)), "state_has_stickiness"),
        (dict(has_hier_rules=2), "has_hier_rules is neither"),
    ]
    for o, msg in cases:
        with pytest.raises(blance_b200.BlanceError, match="scenario 1: .*" + msg):
            ctx.plan_scenarios(t, scs, False, opts=[{}, o])
    # an unknown group bit, through the raw struct
    base = t.struct()
    arr = (abi.Scenario * 1)()
    rm, ad = np.zeros(t.n_node_ids, np.uint8), np.zeros(t.n_node_ids, np.uint8)
    arr[0].node_removed, arr[0].node_added = rm.ctypes.data, ad.ctypes.data
    bad = (abi.ScenarioOpts * 1)()
    bad[0].set = 16
    outs = (abi.ScenarioOut * 1)()
    assert ctx.lib.blance_plan_scenarios_ex(ctx.ptr, ctypes.byref(base), 1, arr, bad, 0, 0, outs) == -1
    assert b"unknown bit" in ctx.lib.blance_last_error(ctx.ptr)
    check_against_oracle(ctx, t, scs, [{}, random_option(t, rng)], False)
