"""blance_plan_scenarios_schedule on the device: every (scenario, count) summary EQUALS the helper of
test_scenario_schedule applied to the serial oracle (tests/schedule_oracle.c) on the fast oracle's move lists of
that scenario's rows, and blance_moves_create + blance_moves_schedule on the same rows; the plans equal
blance_plan_scenarios_ex's; nothing depends on the wave, the engine, the order of the counts or the devices.  Needs
an H100; run with -m gpu."""
import ctypes

import numpy as np
import pytest

import schedule_oracle as SO
from test_scenario_schedule import assert_same_summaries, schedule_summaries
from test_scenarios_gpu import FAST, _fresh_then_rebalance, _node_failures, _same_results, random_base, random_scenarios

import blance_b200
from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu
COUNTS = [-1, 0, 1, 2, 3, 7, 64]


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def move_lists(t, next_rows, favor):
    """CSR move lists of every partition (fast oracle): assigned ones from the pristine prev row (empty when absent
    from prevMap) to the next row, no ops for the others.  Also the beg / end rows that give the same lists."""
    assigned = t.part_in_assign != 0
    beg = np.where(((t.part_in_prev != 0) & assigned)[:, None], t.prev_rows, -1).astype(np.int32)
    end = np.ascontiguousarray(next_rows, np.int32).copy()
    beg[~assigned] = end[~assigned]
    P, SL = t.n_parts, t.n_slots
    max_ops = max(1, 2 * SL)
    node = np.zeros((max(P, 1), max_ops), np.int32)
    state = np.zeros((max(P, 1), max_ops), np.uint8)
    kind = np.zeros((max(P, 1), max_ops), np.uint8)
    cnt = np.zeros(max(P, 1), np.int32)
    slot_off = np.ascontiguousarray(t.state_slot_off, np.int32)
    if P:
        assert FAST.oracle_fast_calc_partition_moves(P, t.n_states, t.n_states, slot_off.ctypes.data, np.ascontiguousarray(beg).ctypes.data,
                                                     end.ctypes.data, int(favor), max_ops, node.ctypes.data, state.ctypes.data,
                                                     kind.ctypes.data, cnt.ctypes.data) == 0
    cnt = cnt[:P]
    valid = np.arange(max_ops)[None, :] < cnt[:, None]
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    return off, node[:P][valid], kind[:P][valid], beg, end


def got_summaries(s):
    return dict(rounds=s.rounds, moves_done=s.moves_done, stuck_parts=s.stuck_parts, max_batch=s.max_batch,
                node_rounds=s.node_rounds, node_last_round=s.node_last_round, part_done_round=s.part_done_round)


def default_mover(t):
    return (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8)


def check_schedules(ctx, base, scs, favor, counts=COUNTS, opts=None, mover=None, with_moves_schedule=True, **kw):
    """Plans + schedules in one call; every (scenario, count) against the serial oracle and, when asked, against
    blance_moves_create + blance_moves_schedule; plans against blance_plan_scenarios_ex."""
    res = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), opts=opts, schedule=counts, node_has_mover=mover, **kw)
    plain = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), opts=opts if opts is not None else [{} for _ in scs], **kw)
    _same_results(res, plain)
    mv = default_mover(base) if mover is None else np.asarray(mover, np.uint8)
    for i, (sc, r) in enumerate(zip(scs, res)):
        t = tables.scenario_tables(base, sc, None if opts is None else opts[i])
        off, node, kind, beg, end = move_lists(t, r.next_rows, favor)
        assert int(off[-1]) == r.ops_total
        h = ctx.moves_create(t.state_slot_off, beg, end, favor, t.n_node_ids)[0] if with_moves_schedule else None
        for c, s in zip(counts, r.schedules):
            ro, so, _ = SO.schedule(off, node, kind, t.n_node_ids, c, mv)
            want = schedule_summaries(off, node, t.n_node_ids, ro, so)
            assert_same_summaries(got_summaries(s), want, (i, c))
            if h is not None:
                d_ro, d_so, _ = ctx.moves_schedule(h, c, mv)
                assert_same_summaries(got_summaries(s), schedule_summaries(off, node, t.n_node_ids, d_ro, d_so), (i, c, "device"))
        if h is not None:
            ctx.moves_free(h)
    return res


@pytest.mark.parametrize("chunk", range(3))
def test_random_scenarios_equal_the_oracle(ctx, chunk):
    for seed in range(chunk * 5, (chunk + 1) * 5):
        t, rng = random_base(seed)
        if t.part_in_assign.all() and rng.random() < 0.5:
            t.part_in_prev[:int(t.n_parts // 10)] = 0
            t.prev_rows[:int(t.n_parts // 10)] = -1
            t.prev_shape[:int(t.n_parts // 10)] = 0
        scs = random_scenarios(t, rng, int(rng.integers(1, 7)))
        if not t.part_in_prev.all():
            for sc in scs:
                sc["node_removed"][:] = 0
        check_schedules(ctx, t, scs, bool(seed % 2))


def test_option_scenarios_equal_the_oracle(ctx):
    t, rng = random_base(41)
    w = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
    S = w.n_states
    opts = [{}, dict(state_constraints=np.asarray(w.state_constraints, np.int32) + 1),
            dict(state_stickiness=np.full(S, 3, np.int32), state_has_stickiness=np.ones(S, np.uint8)),
            dict(state_stickiness=np.zeros(S, np.int32), state_has_stickiness=np.ones(S, np.uint8))]
    scs = random_scenarios(w, rng, len(opts))
    check_schedules(ctx, w, scs, False, counts=[1, 2, 64], opts=opts)


@pytest.mark.parametrize("cfg,P", [(1, 2048), (2, None), (3, 4096)])
def test_synthetic_configurations(ctx, cfg, P):
    size = {} if P is None else dict(P=P)
    t = _fresh_then_rebalance(ctx, cfg, **size) if cfg != 1 else synth.make_fresh(1, **size)
    scs = _node_failures(t, [[], [0], [1, 2]]) + [dict(node_added=(np.arange(t.n_node_ids) < 2).astype(np.uint8))]
    check_schedules(ctx, t, scs, False, counts=[1, 2, 4])


def test_cfg4_reduced(ctx):
    t = synth.make_rebalance(4, P=16384)
    check_schedules(ctx, t, _node_failures(t, [[j] for j in range(4)]), False, counts=[1, 4], with_moves_schedule=False)


def _flat(res):
    return [[(s.rounds, s.moves_done, s.stuck_parts, s.max_batch, s.node_rounds.tobytes(), s.node_last_round.tobytes(),
              s.part_done_round.tobytes()) for s in r.schedules] for r in res]


def test_results_do_not_depend_on_wave_engine_order_or_devices(ctx):
    t, rng = random_base(7)
    scs = random_scenarios(t, rng, 5)
    counts = [1, 3, 2]
    first = _flat(ctx.plan_scenarios(t, scs, False, schedule=counts))
    for mc in (1, 2, 0):
        assert _flat(ctx.plan_scenarios(t, scs, False, max_concurrent=mc, schedule=counts)) == first
    for i in range(len(scs)):                                   # a lone scenario
        assert _flat(ctx.plan_scenarios(t, [scs[i]], False, schedule=counts)) == [first[i]]
    t.engine = 1
    assert _flat(ctx.plan_scenarios(t, scs, False, schedule=counts)) == first
    t.engine = 0
    other = _flat(ctx.plan_scenarios(t, scs, False, schedule=[2, 1, 1, 3, 2]))
    assert [[r[1], r[3], r[0]] for r in other] == first and all(r[2] == r[1] and r[4] == r[0] for r in other)
    import torch
    multi = tables.Context(device_ids=list(range(torch.cuda.device_count())))
    try:
        assert _flat(multi.plan_scenarios(t, scs, False, schedule=counts)) == first
    finally:
        multi.close()


def test_movers(ctx):
    seed = next(x for x in range(100) if (lambda b: b.n_node_ids > b.n_nodes and b.part_in_assign[1])(random_base(x)[0]))
    t, rng = random_base(seed)                                # prev row 1 holds a name outside nodesAll
    scs = random_scenarios(t, rng, 3)
    res = check_schedules(ctx, t, scs, False, counts=[1, 2])
    assert any(s.stuck_parts > 0 for r in res for s in r.schedules)
    mover = default_mover(t)
    mover[rng.permutation(t.n_nodes)[:3]] = 0
    check_schedules(ctx, t, scs, False, counts=[1, 2], mover=mover)
    res = ctx.plan_scenarios(t, scs, False, schedule=[1, 2], node_has_mover=np.zeros(t.n_node_ids, np.uint8))
    for r in res:
        for s in r.schedules:
            assert s.rounds == 0 and s.moves_done == 0 and s.stuck_parts == r.parts_moved
            assert (s.part_done_round != 0).sum() == r.parts_moved and (s.part_done_round <= 0).all()


def test_edges(ctx):
    rng = np.random.default_rng(5)
    # a scenario with no ops
    t = tables.PlanTables(6, 1, 40, [0], [2])
    rows = np.stack([rng.permutation(6)[:2] for _ in range(40)]).astype(np.int32)
    t.prev_rows[:] = rows; t.cur_rows[:] = rows
    t.prev_shape[:] = 2; t.cur_shape[:] = 2; t.part_in_prev[:] = 1
    t.part_in_assign[:] = 0
    res = check_schedules(ctx, t, [{}], False)
    assert res[0].ops_total == 0 and all(s.rounds == 0 for s in res[0].schedules)
    # n_parts tiny
    tiny = tables.PlanTables(5, 1, 1, [0], [2])
    tiny.part_in_prev[:] = 0; tiny.prev_shape[:] = 0
    check_schedules(ctx, tiny, [{}, dict(node_removed=np.array([1, 0, 0, 0, 0], np.uint8))], False)
    # one node with thousands of entries: every partition moves onto node 0
    P = 6000
    big = tables.PlanTables(41, 1, P, [0], [1])
    big.prev_rows[:, 0] = 1 + np.arange(P) % 40
    big.cur_rows[:] = big.prev_rows
    big.prev_shape[:] = 2; big.cur_shape[:] = 2; big.part_in_prev[:] = 1
    rm = np.ones(41, np.uint8); rm[0] = 0
    res = check_schedules(ctx, big, [dict(node_removed=rm)], False, counts=[1, 64], with_moves_schedule=False)
    assert res[0].schedules[1].max_batch == 64
    # 8 192 node ids
    wide = synth.make_rebalance(4, P=4096, N=8192)
    assert wide.n_node_ids >= 8192
    check_schedules(ctx, wide, _node_failures(wide, [[3]]), False, counts=[1, 3], with_moves_schedule=False)


def test_argument_errors(ctx):
    t, rng = random_base(3)
    with pytest.raises(blance_b200.BlanceError, match="scenario 1: add_is_nil"):
        ctx.plan_scenarios(t, [{}, {"add_is_nil": 2}], False, schedule=[1])
    with pytest.raises(blance_b200.BlanceError, match="n_move_conc"):
        ctx.plan_scenarios(t, [{}], False, schedule=[])
    lib = ctx.lib
    base = t.struct()
    scs = (blance_b200.api.Scenario * 1)()
    outs = (blance_b200.api.ScenarioOut * 1)()
    counts = (ctypes.c_int32 * 1)(1)
    assert lib.blance_plan_scenarios_schedule(ctx.ptr, ctypes.byref(base), 1, scs, None, 0, 0, 1, counts, None, outs, None) == -1
    assert lib.blance_plan_scenarios_schedule(ctx.ptr, ctypes.byref(base), 1, scs, None, 0, 0, 1, None, None, outs, outs) == -1
    check_schedules(ctx, t, random_scenarios(t, rng, 2), False, counts=[1])


def test_no_new_kernel_without_schedules(ctx):
    t, rng = random_base(5)
    scs = random_scenarios(t, rng, 3)
    ctx.plan_scenarios(t, scs, False)
    n0 = ctx.kernel_launches()
    ctx.plan_scenarios(t, scs, False)
    plain = ctx.kernel_launches() - n0
    n0 = ctx.kernel_launches()
    ctx.plan_scenarios(t, scs, False, schedule=[1])
    assert ctx.kernel_launches() - n0 > plain


@pytest.mark.parametrize("c", [1, 4])
def test_full_size_headline_failures(ctx, c):
    t = synth.make_rebalance(4)
    scs = _node_failures(t, [[j] for j in (0, 1, 2, 3)])
    res = ctx.plan_scenarios(t, [dict(sc, node_removed=np.maximum(sc["node_removed"], t.node_removed)) for sc in scs],
                             False, want_rows=range(4), schedule=[c])
    mv = default_mover(t)
    for i, r in enumerate(res):
        off, node, kind, _, _ = move_lists(t, r.next_rows, False)
        ro, so, _ = SO.schedule(off, node, kind, t.n_node_ids, c, mv)
        assert_same_summaries(got_summaries(r.schedules[0]), schedule_summaries(off, node, t.n_node_ids, ro, so), (i, c))
        assert r.schedules[0].moves_done == r.ops_total and r.schedules[0].rounds > 0


def test_host_twin_matches_interned_tables_and_orchestrate_schedule():
    """PlanNextMapScenarios(..., scheduleConcurrency) against the summaries derived on the intern_scenario tables, and,
    on fixed-width names (interning order = byte order), against OrchestrateSchedule(prevMap, next_map) round for
    round: the count of rounds, the batches per node and the last round per node."""
    import random
    import types

    from blance_b200 import _host, api
    rnd = random.Random(17)
    nodes = ["n%02d" % i for i in range(12)]
    model = {"primary": (0, 1), "replica": (1, 1)}
    prev = {}
    for p in range(300):
        a = rnd.sample(nodes, 2)
        prev["p%03d" % p] = {"primary": [a[0]], "replica": [a[1]]}
    scs = [{"nodesToRemove": [nodes[j]], "nodesToAdd": None} for j in range(3)] + [{"nodesToRemove": [], "nodesToAdd": [nodes[0]]}]
    counts = [1, 3]
    res = blance_b200.PlanNextMapScenarios(prev, prev, nodes, model, None, scs, wantMaps=range(len(scs)), scheduleConcurrency=counts)
    for i, r in enumerate(res):
        ip = api.intern_scenario(prev, prev, nodes, model, None, scs, i)
        tb = ip.tables()
        out = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, out.out_ptr) == 0
        P, SL = ip.n_parts, ip.n_slots
        t = types.SimpleNamespace(part_in_assign=np.asarray(tb["part_in_assign"]), part_in_prev=np.asarray(tb["part_in_prev"]),
                                  prev_rows=np.asarray(tb["prev_rows"]).reshape(P, SL), state_slot_off=np.asarray(tb["state_slot_off"]),
                                  n_parts=P, n_slots=SL, n_states=ip.n_states)
        off, node, kind, _, _ = move_lists(t, np.asarray(out.next_rows).reshape(P, SL), False)
        mover = (np.arange(ip.n_node_ids) < ip.n_nodes).astype(np.uint8)
        assert [s["MaxConcurrentPartitionMovesPerNode"] for s in r["schedules"]] == counts
        for c, s in zip(counts, r["schedules"]):
            ro, so, _ = SO.schedule(off, node, kind, ip.n_node_ids, c, mover)
            want = schedule_summaries(off, node, ip.n_node_ids, ro, so)
            assert (s["Rounds"], s["MovesDone"], s["StuckParts"], s["MaxBatch"]) == \
                (want["rounds"], want["moves_done"], want["stuck_parts"], want["max_batch"])
            assert s["NodeRounds"] == {ip.node_names[q]: int(v) for q, v in enumerate(want["node_rounds"]) if v}
            assert s["NodeLastRound"] == {ip.node_names[q]: int(v) for q, v in enumerate(want["node_last_round"]) if v}
            rounds = blance_b200.OrchestrateSchedule(model, blance_b200.OrchestratorOptions(MaxConcurrentPartitionMovesPerNode=c),
                                                     nodes, prev, r["next_map"])
            assert len(rounds) == s["Rounds"]
            per_node, last = {}, {}
            for k, batches in enumerate(rounds):
                for b in batches:
                    per_node[b[0]] = per_node.get(b[0], 0) + 1
                    last[b[0]] = k + 1
            assert per_node == s["NodeRounds"] and last == s["NodeLastRound"]
    plain = blance_b200.PlanNextMapScenarios(prev, prev, nodes, model, None, scs)
    assert all("schedules" not in d for d in plain)
