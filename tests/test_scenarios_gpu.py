"""What-if scenarios of one cluster on the device (blance_plan_scenarios): every scenario's plan equals the CPU
oracle on its substituted tables, every summary equals a reference recomputed on the host, and nothing depends on
the wave size, the engine or the number of devices.  Needs an H100; run with `-m gpu`."""
import copy
import ctypes

import numpy as np
import pytest

import golden_util as G
from oracle_loader import fast_lib_path

import blance_b200
from blance_b200 import synth, tables

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
    """The summaries of blance_plan_scenarios recomputed on the host: CalcPartitionMoves (fast oracle) from the
    pristine prev row (empty when absent from prevMap) to the next row of every assigned partition, and
    countStateNodes over the final map."""
    assigned = t.part_in_assign != 0
    in_prev = t.part_in_prev != 0
    NU, S, SL = t.n_node_ids, t.n_states, t.n_slots
    beg = np.where(in_prev[:, None], t.prev_rows, -1).astype(np.int32)[assigned]
    end = np.ascontiguousarray(next_rows[assigned], np.int32)
    beg = np.ascontiguousarray(beg)
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


def check_against_oracle(ctx, base, scs, favor, **kw):
    res = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), **kw)
    for i, (sc, got) in enumerate(zip(scs, res)):
        t = tables.scenario_tables(base, sc)
        ref = oracle_tables(t)
        assert_scenario(got, ref, reference_summary(t, ref.next_rows, ref.warn, favor), i)
    return res


def random_base(seed):
    """Mid-size random flat instances: churn, weights, stickiness, partial assignment, partitions absent from
    prevMap and a node name outside nodesAll."""
    rng = np.random.default_rng(seed + 1000)
    N = int(rng.integers(6, 160))
    S = int(rng.integers(1, 4))
    k = [int(rng.integers(1, 4)) if s < 2 else int(rng.integers(0, 2)) for s in range(S)]
    while sum(k) > N - 2:
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
    sh = np.full((P, S), 2, np.uint8)
    t.prev_shape[:] = sh
    t.cur_shape[:] = sh
    t.part_in_prev[:] = 1
    if rng.random() < 0.3:
        t.part_in_assign[:] = (rng.random(P) < 0.8).astype(np.uint8)
    if rng.random() < 0.6:
        t.has_part_weights = 1
        t.part_has_weight[:] = (rng.random(P) < 0.4).astype(np.uint8)
        t.part_weight[:] = rng.integers(1, 9, P)
        t.state_has_stickiness[:] = (rng.random(S) < 0.7).astype(np.uint8)
        t.state_stickiness[:] = rng.integers(0, 5, S)
    t.booster_kind = int(rng.random() < 0.3)
    t.max_iters = int(rng.integers(1, 6))
    return t, rng


def random_scenarios(t, rng, count):
    N, NU = t.n_nodes, t.n_node_ids
    # the base's own node fields (ignored by the call) and an identical copy, then random variants
    scs = [dict(node_removed=t.node_removed.copy(), node_added=t.node_added.copy(), add_is_nil=0, has_node_weights=0,
                node_weight=np.zeros(N, np.int32), node_has_weight=np.zeros(N, np.uint8)),
           dict(node_removed=np.ones(NU, np.uint8), node_added=np.zeros(NU, np.uint8), add_is_nil=1, has_node_weights=0,
                node_weight=np.zeros(N, np.int32), node_has_weight=np.zeros(N, np.uint8))]
    while len(scs) < count:
        rm = np.zeros(NU, np.uint8)
        rm[rng.permutation(NU)[:int(rng.integers(0, max(1, N // 6)))]] = 1
        ad = np.zeros(NU, np.uint8)
        ad[rng.permutation(N)[:int(rng.integers(0, N // 4 + 1))]] = 1
        hw = int(rng.random() < 0.5)
        scs.append(dict(node_removed=rm, node_added=ad, add_is_nil=int(rng.random() < 0.15), has_node_weights=hw,
                        node_weight=rng.integers(-2, 7, N).astype(np.int32),
                        node_has_weight=(rng.random(N) < 0.8).astype(np.uint8)))
    return scs[:count]


@pytest.mark.parametrize("chunk", range(5))
def test_random_scenarios_match_oracle_and_reference_summary(ctx, chunk):
    for seed in range(chunk * 8, (chunk + 1) * 8):
        t, rng = random_base(seed)
        if t.part_in_assign.all() and rng.random() < 0.5:
            t.part_in_prev[:int(t.n_parts // 10)] = 0     # partitions new to this map: an empty beg row
            t.prev_rows[:int(t.n_parts // 10)] = -1
            t.prev_shape[:int(t.n_parts // 10)] = 0
        scs = random_scenarios(t, rng, int(rng.integers(1, 13)))
        if not t.part_in_prev.all():                   # plan.go:544: no removal with partitions absent from prevMap
            for sc in scs:
                sc["node_removed"][:] = 0
        check_against_oracle(ctx, t, scs, bool(seed % 2))


def _same_results(a, b):
    for x, y in zip(a, b):
        for f in ("next_rows", "next_shape", "warn", "node_ops", "state_node_load"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), f
        for f in ("iters_run", "converged", "steps", "parts_moved", "ops_total", "warn_parts"):
            assert getattr(x, f) == getattr(y, f), f


def test_results_do_not_depend_on_wave_engine_or_devices(ctx):
    t, rng = random_base(7)
    scs = random_scenarios(t, rng, 7)
    first = ctx.plan_scenarios(t, scs, False, want_rows=range(7))
    for mc in (1, 3, 0):
        _same_results(first, ctx.plan_scenarios(t, scs, False, max_concurrent=mc, want_rows=range(7)))
    for engine in (0, 1, 2):
        t.engine = engine
        _same_results(first, ctx.plan_scenarios(t, scs, False, want_rows=range(7)))
    t.engine = 0
    import torch
    multi = tables.Context(device_ids=list(range(torch.cuda.device_count())))
    try:
        _same_results(first, multi.plan_scenarios(t, scs, False, want_rows=range(7)))
    finally:
        multi.close()


def _fresh_then_rebalance(ctx, cfg, **size):
    fresh = synth.make_fresh(cfg, **size)
    rows = ctx.plan_next_map(fresh).next_rows
    return synth.make_rebalance(cfg, prev_rows=rows, **size)


def _node_failures(t, nodes):
    out = []
    for group in nodes:
        rm = np.zeros(t.n_node_ids, np.uint8)
        rm[list(group)] = 1
        out.append(dict(node_removed=rm, node_added=np.zeros(t.n_node_ids, np.uint8), add_is_nil=0))
    return out


def test_cfg2_every_rack_failure(ctx):
    t = _fresh_then_rebalance(ctx, 2)
    scs = _node_failures(t, [range(r * 8, r * 8 + 8) for r in range(t.n_nodes // 8)])
    check_against_oracle(ctx, t, scs, False)


def test_cfg4_reduced_single_node_failures(ctx):
    t = synth.make_rebalance(4, P=16384)
    scs = _node_failures(t, [[j] for j in range(8)])
    res = check_against_oracle(ctx, t, scs, False)
    assert all(r.sticky_steps > 0 for r in res)          # the speculative kernel ran inside the wave


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_string_api_own_node_sets(c):
    kw = G.plan_kwargs(c)
    prev = kw["prev_map"]
    assign = kw["partitions_to_assign"] if kw["partitions_to_assign"] is not None else prev
    before = (copy.deepcopy(prev), copy.deepcopy(assign))
    o = blance_b200.PlanNextMapOptions(
        ModelStateConstraints=kw["model_state_constraints"], PartitionWeights=kw["partition_weights"],
        StateStickiness=kw["state_stickiness"], NodeWeights=kw["node_weights"], NodeHierarchy=kw["node_hierarchy"],
        HierarchyRules=kw["hierarchy_rules"], NodeScoreBooster=kw["booster"])
    r = blance_b200.PlanNextMapScenarios(prev, assign, kw["nodes_all"], kw["model"], o,
                                         [{"nodesToRemove": kw["nodes_to_remove"], "nodesToAdd": kw["nodes_to_add"]}],
                                         wantMaps=[0])
    assert r[0]["next_map"] == G.pmap(c["exp"])
    assert G.count_warnings(c, r[0]["warnings"]) == c["expNumWarnings"]
    assert (prev, assign) == before                      # no side effects on the caller's maps


def test_errors_leave_the_context_usable(ctx):
    t, rng = random_base(3)
    lib = ctx.lib
    base = t.struct()
    outs = (blance_b200.api.ScenarioOut * 1)()
    scs = (blance_b200.api.Scenario * 1)()
    assert lib.blance_plan_scenarios(ctx.ptr, ctypes.byref(base), 0, scs, 0, 0, outs) == -1
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: add_is_nil"):
        ctx.plan_scenarios(t, [{}, {"add_is_nil": 2}], False)
    check_against_oracle(ctx, t, random_scenarios(t, rng, 2), False)
