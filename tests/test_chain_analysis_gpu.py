"""blance_plan_chains_exposure on the device: plans and nets equal blance_plan_chains; every stage's schedule, audit and
exposure equals the handle path (blance_moves_create -> _schedule -> _exposure) and blance_map_audit on that stage's
maps; the net rebalance equals the handle path from the base's prev rows to the last stage's map; the span equals the
CPU reference (tests/chain_analysis_ref.py) and does not depend on the per-stage arrays, the wave size, the engine or
the number of devices.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import chain_analysis_ref as CA
import chain_util as C
import exposure_oracle as EO
import scenario_exposure_ref as REF
from test_chains_gpu import random_chains
from test_scenario_audit_gpu import _forest, final_map, flat
from test_scenario_exposure_gpu import _tiny_base, handle_exposure
from test_scenario_schedule import schedule_summaries
from test_scenarios_gpu import _fresh_then_rebalance, _same_results, random_base

from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu
COUNTS = (1, 3)
BIG = 1 << 15


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def handle_schedule(ctx, t, next_rows, favor, count):
    """The schedule summaries of blance_moves_create -> blance_moves_schedule on the handle of the rebalance of tables t
    (begMap partitions), part_done_round scattered to [n_parts]."""
    member, beg, end = REF.begmap_rows(t, next_rows)
    h, total = ctx.moves_create(t.state_slot_off, beg, end, favor, t.n_node_ids)
    off, node, _, _ = ctx.moves_fetch(h, total)
    ro, so, _ = ctx.moves_schedule(h, count, (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8))
    ctx.moves_free(h)
    s = schedule_summaries(off, node, t.n_node_ids, ro, so)
    full = np.zeros(t.n_parts, np.int32)
    full[member] = s["part_done_round"]
    s["part_done_round"] = full
    return s


def same_schedule(got, want, what):
    g = summaries(got)
    for f, v in want.items():
        assert np.array_equal(g[f], v), (what, f)


def summaries(s):
    return dict(rounds=s.rounds, moves_done=s.moves_done, stuck_parts=s.stuck_parts, max_batch=s.max_batch, node_rounds=s.node_rounds,
                node_last_round=s.node_last_round, part_done_round=s.part_done_round)


def same_span(a, b, what):
    assert set(a) == set(b), what
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (what, k)


def run(ctx, base, chains, favor, opts=None, parent=None, **kw):
    T = len(chains[0])
    return ctx.plan_chains(base, chains, favor, want_rows=[(i, t) for i in range(len(chains)) for t in range(T)], opts=opts,
                           schedule=list(COUNTS), audit=dict(n2n=True, domain_parent=parent),
                           exposure=dict(series_cap=BIG, domain_parent=parent), span=True, **kw)


def check(ctx, base, chains, favor, opts=None, parent=None, reference=True, handle=True):
    """Everything of one call against blance_plan_chains, the handle path, blance_map_audit and the CPU reference."""
    T = len(chains[0])
    res, nets, spans = run(ctx, base, chains, favor, opts, parent)
    plain, pnets = ctx.plan_chains(base, chains, favor, want_rows=[(i, t) for i in range(len(chains)) for t in range(T)], opts=opts)
    for i, chain in enumerate(chains):
        _same_results(res[i], plain[i])
        assert np.array_equal(nets[i].node_ops, pnets[i].node_ops)
        assert (nets[i].ops_total, nets[i].parts_moved) == (pnets[i].ops_total, pnets[i].parts_moved)
        o = None if opts is None else opts[i]
        cur = base
        for t, stage in enumerate(chain):
            x = C.substituted(cur, stage, o, t)
            r = res[i][t]
            rows, shape = final_map(x, r)
            assert flat(r.audit) == flat(ctx.map_audit(x, rows, shape, n2n=True, domain_parent=parent)), (i, t)
            for k, c in enumerate(COUNTS):
                assert r.exposures[k]["rounds"] == r.schedules[k].rounds
                if handle:
                    same_schedule(r.schedules[k], handle_schedule(ctx, x, r.next_rows, favor, c), (i, t, c, "handle"))
                    EO.assert_equal(r.exposures[k], handle_exposure(ctx, x, r.next_rows, favor, c, parent), (i, t, c, "handle"))
            cur = C.advance(cur, r.next_rows, r.next_shape)
        xn = C.substituted(base, chain[-1], o, 0)
        for k, c in enumerate(COUNTS):
            assert nets[i].exposures[k]["rounds"] == nets[i].schedules[k].rounds
            if handle:
                same_schedule(nets[i].schedules[k], handle_schedule(ctx, xn, res[i][-1].next_rows, favor, c), (i, c, "net"))
                EO.assert_equal(nets[i].exposures[k], handle_exposure(ctx, xn, res[i][-1].next_rows, favor, c, parent), (i, c, "net"))
            # the span is the numpy fold of the per-stage outputs
            want = CA.fold([summaries(res[i][t].schedules[k]) for t in range(T)], [res[i][t].exposures[k] for t in range(T)])
            CA.assert_span(spans[i][k], want, (i, c, "fold"))
        if reference:
            stages, net, rspans = CA.chain_analysis(base, chain, o, favor, COUNTS, domain_parent=parent)
            for t in range(T):
                for k, c in enumerate(COUNTS):
                    for f, v in stages[t][k][0].items():
                        assert np.array_equal(summaries(res[i][t].schedules[k])[f], v), (i, t, c, f)
                    EO.assert_equal(res[i][t].exposures[k], stages[t][k][1], (i, t, c, "reference"))
            for k, c in enumerate(COUNTS):
                for f, v in net[k][0].items():
                    assert np.array_equal(summaries(nets[i].schedules[k])[f], v), (i, c, "net", f)
                EO.assert_equal(nets[i].exposures[k], net[k][1], (i, c, "net reference"))
                CA.assert_span(spans[i][k], rspans[k], (i, c, "span reference"))
    # the span alone: no per-stage array asked for, the same span
    _, _, alone = run(ctx, base, chains, favor, opts, parent, stage_arrays=False)
    for i in range(len(chains)):
        for k in range(len(COUNTS)):
            same_span(alone[i][k], spans[i][k], (i, k, "span alone"))
    return res, nets, spans


def same_all(a, b, what):
    (ra, na, sa), (rb, nb, sb) = a, b
    for i in range(len(ra)):
        _same_results(ra[i], rb[i])
        for x, y in zip(ra[i], rb[i]):
            for s, q in zip(x.schedules, y.schedules):
                for f, v in summaries(s).items():
                    assert np.array_equal(v, summaries(q)[f]), (what, f)
            assert flat(x.audit) == flat(y.audit), what
            for e, g in zip(x.exposures, y.exposures):
                EO.assert_equal(e, g, what)
        for e, g in zip(na[i].exposures, nb[i].exposures):
            EO.assert_equal(e, g, what)
        for s, q in zip(sa[i], sb[i]):
            same_span(s, q, what)


def test_random_chains(ctx):
    for seed in (2, 9, 23):
        t, rng = random_base(seed)
        check(ctx, t, random_chains(t, rng, 3, 1 + seed % 3), bool(seed % 2))


def test_raised_constraints_and_forest(ctx):
    t, rng = random_base(41)
    w = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
    opts = [{}, dict(state_constraints=np.asarray(w.state_constraints, np.int32) + 1), {}]
    from test_exposure_oracle import random_forest
    check(ctx, w, random_chains(w, rng, 3, 3), False, opts=opts, parent=random_forest(rng, w.n_node_ids, 3))


def test_one_stage_equals_scenarios_exposure(ctx):
    t, rng = random_base(7)
    chains = [[dict(st, node_in_all=np.ones(t.n_nodes, np.uint8))] for st in (c[0] for c in random_chains(t, rng, 4, 1))]
    res, nets, spans = run(ctx, t, chains, True)
    scs = [{k: v for k, v in c[0].items() if k != "node_in_all"} for c in chains]
    want = ctx.plan_scenarios(t, scs, True, want_rows=range(len(scs)), schedule=list(COUNTS), audit=dict(n2n=True),
                              exposure=dict(series_cap=BIG))
    for i, w in enumerate(want):
        r = res[i][0]
        _same_results([r], [w])
        assert flat(r.audit) == flat(w.audit)
        for k in range(len(COUNTS)):
            assert summaries(r.schedules[k]).keys() == summaries(w.schedules[k]).keys()
            for f, v in summaries(r.schedules[k]).items():
                assert np.array_equal(v, summaries(w.schedules[k])[f]), f
            EO.assert_equal(r.exposures[k], w.exposures[k], (i, k))
            sp, e, s = spans[i][k], w.exposures[k], w.schedules[k]
            assert (sp["rounds"], sp["moves_done"], sp["stuck_parts"], sp["max_batch"]) == (s.rounds, s.moves_done, s.stuck_parts, s.max_batch)
            assert np.array_equal(sp["part_done_round"], s.part_done_round) and np.array_equal(sp["node_last_round"], s.node_last_round)
            for f in ("peak", "peak_round", "area", "part_min_copies", "part_no_top", "part_flags", "dom_peak", "dom_peak_round"):
                assert np.array_equal(sp[f], e[f]), f
            assert not sp["peak_stage"].any() and not sp["dom_peak_stage"].any()


def test_no_dependence_on_wave_engine_or_devices(ctx):
    t, rng = random_base(11)
    chains = random_chains(t, rng, 5, 3)
    first = run(ctx, t, chains, False)
    for engine in (0, 1, 2):
        t.engine = engine
        for mc in (1, 3, 0) if engine == 0 else (0,):
            same_all(run(ctx, t, chains, False, max_concurrent=mc), first, (engine, mc))
    t.engine = 0
    multi = tables.Context(device_ids=[0])
    try:
        same_all(run(multi, t, chains, False), first, "multi")
    finally:
        multi.close()


def _rolling_upgrade(t, nodes):
    """One chain per node: remove it, then add it back (it stays in nodesAll: the removal already stripped it)."""
    chains = []
    for q in nodes:
        rm, ad = np.zeros(t.n_node_ids, np.uint8), np.zeros(t.n_node_ids, np.uint8)
        rm[q], ad[q] = 1, 1
        every = np.ones(t.n_nodes, np.uint8)
        chains.append([dict(node_removed=rm, node_in_all=every), dict(node_added=ad, node_in_all=every)])
    return chains


def test_cfg2_rack_forest(ctx):
    t = _fresh_then_rebalance(ctx, 2)
    check(ctx, t, _rolling_upgrade(t, [0, 5, 17]), False, parent=_forest(t, 2), reference=False)


def test_cfg4_reduced_rolling_upgrade(ctx):
    t = synth.make_rebalance(4, P=16384)
    check(ctx, t, _rolling_upgrade(t, [0, 1]), True, reference=False)


def test_more_than_65535_chain_count_pairs(ctx):
    """8 200 chains x 8 counts = 65 600 (chain, count) pairs in one wave: the fold's flat index covers all of them, and
    chains on both sides of 65 535 equal the same chains run alone."""
    t, rng = _tiny_base(3)
    counts = list(range(1, 9))
    chains = []
    for j in range(8200):
        rm = np.zeros(t.n_node_ids, np.uint8)
        rm[int(rng.integers(0, t.n_nodes - 2))] = 1
        ad = np.zeros(t.n_node_ids, np.uint8)
        ad[t.n_nodes - 1 - j % 2] = 1
        chains.append([dict(node_removed=rm, add_is_nil=0), dict(node_added=ad, add_is_nil=0)])
    kw = dict(schedule=counts, exposure=dict(series_cap=4), span=True)
    _, _, big = ctx.plan_chains(t, chains, False, **kw)
    sample = [0, 1, 8190, 8191, 8192, 8199]
    _, _, alone = ctx.plan_chains(t, [chains[j] for j in sample], False, **kw)
    moved = 0
    for j, a in zip(sample, alone):
        for x, y in zip(big[j], a):
            same_span(x, y, j)
            moved += int(x["rounds"] > 0)
    assert moved > 0


# kernels launched by the second of two identical blance_plan_chains calls on random_base(5), 3 chains of 2 stages,
# max_concurrent = 3, counted with the build before blance_plan_chains_exposure existed
PARENT_CHAIN_LAUNCHES = 145


def test_plan_chains_launches_as_before(ctx):
    t, rng = random_base(5)
    chains = random_chains(t, rng, 3, 2)

    def launches(**kw):
        ctx.plan_chains(t, chains, False, max_concurrent=3, **kw)
        n0 = ctx.kernel_launches()
        ctx.plan_chains(t, chains, False, max_concurrent=3, **kw)
        return ctx.kernel_launches() - n0
    before = launches()
    assert before == PARENT_CHAIN_LAUNCHES
    launches(schedule=[1], exposure={}, span=True)
    assert launches() == before                     # an analysis leaves nothing behind that changes a later plain call
