"""blance_plan_chains_ex on the device: chains whose stages set plan options of their own.  The same options at every
stage equal blance_plan_chains_exposure byte for byte with as many kernel launches; one stage equals
blance_plan_scenarios_exposure; per-stage options equal the per-stage CPU reference (tests/chain_stage_util.py) and,
per stage, the handle path and blance_map_audit on that stage's maps under that stage's options, whatever the wave size,
engine or context; the string face equals the literal oracle driven as the Go loop; and the chain entry points without
per-stage options launch as many kernels as before.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import chain_analysis_ref as CA
import chain_stage_util as CS
import chain_util as C
import exposure_oracle as EO
from randgen import random_instance
from test_chain_analysis_gpu import handle_schedule, same_all, same_span, summaries
from test_chains import make_chain
from test_chains_gpu import random_chains
from test_exposure_oracle import random_forest
from test_scenario_audit_gpu import final_map, flat
from test_scenario_exposure_gpu import handle_exposure
from test_scenario_options import options_of
from test_scenario_options_gpu import rack_masks, random_base, random_option
from test_scenarios import removal_allowed
from test_scenarios_gpu import _same_results

import blance_b200
from blance_b200 import tables

pytestmark = pytest.mark.gpu
COUNTS = (1, 3)
BIG = 1 << 15


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def staged_options(t, rng, n, T, kind=None):
    """[n][T] option dicts over tables t (slot ranges one wider than the constraints), one pattern per chain:
    0  the first state's constraint raised at stage 1 and back to the base's after it (1 -> 2 -> 1 from a base of 1);
    1  stickiness changed at one stage only;
    2  weights overridden at stage 0 (presence switched on and off), back to the base's at stage 1, then off at stage 2;
    3  hierarchy rules off at stage 0, first on at the last stage with a wider mask (two rules, from a third stage on);
    4  a random option dict per stage."""
    S = t.n_states
    out = []
    for i in range(n):
        k = (i if kind is None else kind) % 5
        so = [{} for _ in range(T)]
        if k == 0:
            c = np.array(t.state_constraints, np.int32)
            c[0] += 1
            so[min(1, T - 1)] = dict(state_constraints=c)
        elif k == 1:
            so[int(rng.integers(T))] = dict(state_stickiness=rng.integers(0, 9, S).astype(np.int32),
                                            state_has_stickiness=(rng.random(S) < 0.7).astype(np.uint8))
        elif k == 2:
            has = np.flatnonzero(np.asarray(t.part_has_weight) != 0)[:5]
            lacks = np.flatnonzero(np.asarray(t.part_has_weight) == 0)[:5]
            part = np.concatenate([has, lacks]).astype(np.int32)
            so[0] = dict(has_part_weights=1, weight_overrides=(part, rng.integers(1, 30, part.size).astype(np.int32),
                                                                (np.arange(part.size) >= has.size).astype(np.uint8)))
            if T > 2:
                so[2] = dict(has_part_weights=0)
        elif k == 3 and S > 1:
            so[0] = dict(has_hier_rules=0)
            rule_off, mask, R = rack_masks(t, 2, {1} if T < 3 else {0, 1})
            so[T - 1] = dict(has_hier_rules=1, rule_off=rule_off, ie_mask=mask, n_rules=R, n_hier_bits=t.n_nodes)
            if T > 2:
                rule_off, mask, R = rack_masks(t, 4, {1})
                so[1] = dict(has_hier_rules=1, rule_off=rule_off, ie_mask=mask, n_rules=R, n_hier_bits=t.n_nodes)
        else:
            so = [random_option(t, rng) for _ in range(T)]
        out.append(so)
    return out


def check_staged(ctx, base, chains, sopts, favor, parent=None, audit=True, expo=True, reference=True, **kw):
    """One blance_plan_chains_ex call against the per-stage CPU reference, the handle path and blance_map_audit per
    stage, the handle path for the net rebalance (the last stage's constraints) and the fold of the span."""
    n, T = len(chains), len(chains[0])
    args = dict(want_rows=[(i, t) for i in range(n) for t in range(T)], stage_opts=sopts, schedule=list(COUNTS), span=True, **kw)
    if audit:
        args["audit"] = dict(n2n=True, domain_parent=parent)
    if expo:
        args["exposure"] = dict(series_cap=BIG, domain_parent=parent)
    res, nets, spans = ctx.plan_chains(base, chains, favor, **args)
    for i, chain in enumerate(chains):
        if reference:
            ref, rnet = CS.chain_reference_staged(base, chain, sopts[i], favor)
            for t in range(T):
                C.assert_stage(res[i][t], ref[t], (i, t))
            assert np.array_equal(nets[i].node_ops, rnet["node_ops"]), i
            assert (nets[i].ops_total, nets[i].parts_moved) == (rnet["ops_total"], rnet["parts_moved"]), i
        cur = base
        for t, stage in enumerate(chain):
            x = C.substituted(cur, stage, sopts[i][t], t)
            r = res[i][t]
            if audit:
                rows, shape = final_map(x, r)
                assert flat(r.audit) == flat(ctx.map_audit(x, rows, shape, n2n=True, domain_parent=parent)), (i, t)
            for k, c in enumerate(COUNTS):
                want = handle_schedule(ctx, x, r.next_rows, favor, c)
                for f, v in want.items():
                    assert np.array_equal(summaries(r.schedules[k])[f], v), (i, t, c, f)
                if expo:
                    EO.assert_equal(r.exposures[k], handle_exposure(ctx, x, r.next_rows, favor, c, parent), (i, t, c))
            cur = C.advance(cur, r.next_rows, r.next_shape)
        xn = C.substituted(base, chain[-1], sopts[i][-1], 0)        # the net rebalance: the last stage's constraints
        for k, c in enumerate(COUNTS):
            for f, v in handle_schedule(ctx, xn, res[i][-1].next_rows, favor, c).items():
                assert np.array_equal(summaries(nets[i].schedules[k])[f], v), (i, c, "net", f)
            if expo:
                EO.assert_equal(nets[i].exposures[k], handle_exposure(ctx, xn, res[i][-1].next_rows, favor, c, parent), (i, c, "net"))
                want = CA.fold([summaries(res[i][t].schedules[k]) for t in range(T)], [res[i][t].exposures[k] for t in range(T)])
                CA.assert_span(spans[i][k], want, (i, c, "fold"))
    return res, nets, spans


def _launches(ctx, f):
    f()
    n0 = ctx.kernel_launches()
    r = f()
    return ctx.kernel_launches() - n0, r


# ---- 1. the same options at every stage: blance_plan_chains_exposure byte for byte, as many launches -------------

def test_same_options_every_stage_equal_chains_exposure(ctx):
    t, rng = random_base(41)
    T = 3
    chains = random_chains(t, rng, 5, T)
    opts = [{}, random_option(t, rng), dict(state_constraints=np.asarray(t.state_constraints, np.int32) + 1),
            dict(has_part_weights=1, weight_overrides=(np.arange(0, t.n_parts, 7, dtype=np.int32),
                                                       np.full(len(range(0, t.n_parts, 7)), 5, np.int32),
                                                       (np.arange(len(range(0, t.n_parts, 7))) % 2).astype(np.uint8))),
            random_option(t, rng)]
    staged = [[o] * T for o in opts]
    parent = random_forest(rng, t.n_node_ids, 3)
    want_rows = [(i, s) for i in range(len(chains)) for s in range(T)]
    kw = dict(want_rows=want_rows, schedule=list(COUNTS), audit=dict(n2n=True, domain_parent=parent),
              exposure=dict(series_cap=BIG, domain_parent=parent), span=True, max_concurrent=3)
    la, a = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, opts=opts, **kw))
    lb, b = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=staged, **kw))
    same_all(a, b, "exposure")
    for x, y in zip(a[1], b[1]):
        assert np.array_equal(x.node_ops, y.node_ops) and (x.ops_total, x.parts_moved) == (y.ops_total, y.parts_moved)
        for s, q in zip(x.schedules, y.schedules):
            for f, v in summaries(s).items():
                assert np.array_equal(v, summaries(q)[f]), f
    assert la == lb, (la, lb)          # (sticky_steps counts what the engine did, as in the scenario tests: not compared)
    # without a schedule: blance_plan_chains
    lp, p = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, opts=opts, want_rows=want_rows))
    lq, q = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=staged, want_rows=want_rows))
    for i in range(len(chains)):
        _same_results(p[0][i], q[0][i])
        assert np.array_equal(p[1][i].node_ops, q[1][i].node_ops) and p[1][i].ops_total == q[1][i].ops_total
    assert lp == lq, (lp, lq)


# ---- 2. one stage: blance_plan_scenarios_exposure -----------------------------------------------------------------

def test_one_stage_equals_scenarios_exposure(ctx):
    t, rng = random_base(7)
    chains = [[dict(st, node_in_all=np.ones(t.n_nodes, np.uint8))] for st in (c[0] for c in random_chains(t, rng, 5, 1))]
    opts = [random_option(t, rng) for _ in chains]
    res, nets, spans = ctx.plan_chains(t, chains, True, want_rows=[(i, 0) for i in range(len(chains))], stage_opts=[[o] for o in opts],
                                       schedule=list(COUNTS), audit=dict(n2n=True), exposure=dict(series_cap=BIG), span=True)
    scs = [{k: v for k, v in c[0].items() if k != "node_in_all"} for c in chains]
    want = ctx.plan_scenarios(t, scs, True, want_rows=range(len(scs)), opts=opts, schedule=list(COUNTS), audit=dict(n2n=True),
                              exposure=dict(series_cap=BIG))
    for i, w in enumerate(want):
        r = res[i][0]
        _same_results([r], [w])
        assert flat(r.audit) == flat(w.audit)
        for k in range(len(COUNTS)):
            for f, v in summaries(r.schedules[k]).items():
                assert np.array_equal(v, summaries(w.schedules[k])[f]), f
            EO.assert_equal(r.exposures[k], w.exposures[k], (i, k))


# ---- 3. per-stage options against the CPU reference ---------------------------------------------------------------

@pytest.mark.parametrize("seed", (2, 9, 23, 30))
def test_random_staged_chains(ctx, seed):
    t, rng = random_base(seed)
    T = 2 + seed % 2
    chains = random_chains(t, rng, 5, T)
    check_staged(ctx, t, chains, staged_options(t, rng, 5, T), bool(seed % 2), parent=random_forest(rng, t.n_node_ids, 3))


def test_every_pattern_with_three_stages(ctx):
    t, rng = random_base(3)
    while t.n_states < 2:
        t, rng = random_base(int(rng.integers(100, 10_000)))
    for kind in range(5):
        chains = random_chains(t, rng, 3, 3)
        check_staged(ctx, t, chains, staged_options(t, rng, 3, 3, kind=kind), bool(kind % 2))


def test_analyses_optional(ctx):
    t, rng = random_base(17)
    chains = random_chains(t, rng, 4, 3)
    so = staged_options(t, rng, 4, 3)
    check_staged(ctx, t, chains, so, False, audit=False, expo=False)
    check_staged(ctx, t, chains, so, True, audit=True, expo=False)
    # no schedule at all: the plans alone
    res, nets = ctx.plan_chains(t, chains, False, want_rows=[(i, s) for i in range(4) for s in range(3)], stage_opts=so)
    for i, chain in enumerate(chains):
        ref, rnet = CS.chain_reference_staged(t, chain, so[i], False)
        for s in range(3):
            C.assert_stage(res[i][s], ref[s], (i, s))
        assert nets[i].ops_total == rnet["ops_total"]


def test_no_dependence_on_wave_engine_or_devices(ctx):
    t, rng = random_base(11)
    chains = random_chains(t, rng, 7, 3)
    so = staged_options(t, rng, 7, 3)
    kw = dict(want_rows=[(i, s) for i in range(7) for s in range(3)], stage_opts=so, schedule=list(COUNTS), audit=dict(n2n=True),
              exposure=dict(series_cap=BIG), span=True)
    first = check_staged(ctx, t, chains, so, False, max_concurrent=1)
    for engine in (0, 1, 2):
        t.engine = engine
        for mc in (1, 3, 0) if engine == 0 else (0,):
            same_all(ctx.plan_chains(t, chains, False, max_concurrent=mc, **kw), first, (engine, mc))
    t.engine = 0
    multi = tables.Context(device_ids=[0])
    try:
        same_all(multi.plan_chains(t, chains, False, **kw), first, "multi")
    finally:
        multi.close()


def test_lone_chain_with_a_later_wider_mask(ctx):
    """One chain on the device (the base upload is its plan): the hierarchy masks of a later stage are wider than stage 0's."""
    t, rng = random_base(3)
    while t.n_states < 2:
        t, rng = random_base(int(rng.integers(100, 10_000)))
    chains = random_chains(t, rng, 1, 3)
    check_staged(ctx, t, chains, staged_options(t, rng, 1, 3, kind=3), False)
    check_staged(ctx, t, chains, staged_options(t, rng, 1, 3, kind=2), True)


def test_span_alone_is_the_same(ctx):
    t, rng = random_base(5)
    chains = random_chains(t, rng, 3, 3)
    so = staged_options(t, rng, 3, 3)
    kw = dict(stage_opts=so, schedule=list(COUNTS), exposure=dict(series_cap=BIG), span=True)
    _, _, full = ctx.plan_chains(t, chains, False, **kw)
    _, _, alone = ctx.plan_chains(t, chains, False, stage_arrays=False, **kw)
    for i in range(3):
        for k in range(len(COUNTS)):
            same_span(alone[i][k], full[i][k], (i, k))


# ---- 4. the string face against the literal Go loop --------------------------------------------------------------

def _string_stages(stages, keys):
    out = []
    for (nodes_all, rm, add, nw), k in zip(stages, keys):
        st = dict(k, nodesToRemove=rm, nodesToAdd=add, nodesAll=list(nodes_all))
        if nw != "inherit":
            st["nodeWeights"] = nw
        out.append(st)
    return out


@pytest.mark.parametrize("chunk", range(2))
def test_string_face_equals_literal_loop(chunk):
    checked = 0
    for seed in range(chunk * 30, (chunk + 1) * 30):
        kw = random_instance(seed)
        if not removal_allowed(kw) and kw["nodes_to_remove"]:
            continue
        stages = make_chain(kw, seed)
        if not removal_allowed(kw):
            stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
        keys = CS.make_stage_options(kw, seed, len(stages))
        lit = CS.literal_chain_staged(kw, stages, keys)
        prev, assign = kw["prev_map"], kw["partitions_to_assign"]
        chain = {"stages": _string_stages(stages, keys)}
        res = blance_b200.PlanNextMapChains(prev, prev if assign is None else assign, kw["nodes_all"], kw["model"], options_of(kw),
                                            [chain, chain], seed % 2 == 1, wantMaps=[0])
        for t, l in enumerate(lit):
            r = res[0]["stages"][t]
            assert r["iterations"] == l["iterations"], (seed, t)
            assert r["next_map"] == (l["next_map"] if r["iterations"] > 0 else {}), (seed, t, keys)
            assert r["warnings"] == (l["warnings"] if r["iterations"] > 0 else {}), (seed, t, keys)
            assert res[1]["stages"][t]["ops_total"] == r["ops_total"]
        # with schedules and audits: the same plans
        an = blance_b200.PlanNextMapChains(prev, prev if assign is None else assign, kw["nodes_all"], kw["model"], options_of(kw),
                                           [chain], seed % 2 == 1, wantMaps=[0], scheduleConcurrency=[1, 2], audit={}, exposure={})
        for t in range(len(stages)):
            for f in ("next_map", "warnings", "ops_total", "node_ops", "state_node_load", "iterations"):
                assert an[0]["stages"][t].get(f) == res[0]["stages"][t].get(f), (seed, t, f)
        checked += 1
    assert checked > 10


# ---- 5. the chain entry points without per-stage options launch as before ---------------------------------------

# kernels launched by the second of two identical calls on random_base(5) of tests/test_chains_gpu.py, 3 chains of 2
# stages, max_concurrent = 3, counted with the build before blance_plan_chains_ex: blance_plan_chains (as
# test_chain_analysis_gpu.PARENT_CHAIN_LAUNCHES), and blance_plan_chains_exposure with schedules at counts 1 and 3,
# audits, exposures and spans, and the same with per-chain options that override partition weights
PARENT_LAUNCHES = dict(plain=145, exposure=1329, exposure_weights=1330)


def parent_launch_arms(ctx):
    from test_scenarios_gpu import random_base as base5
    t, rng = base5(5)
    chains = random_chains(t, rng, 3, 2)
    wo = (np.arange(0, t.n_parts, 5, dtype=np.int32), np.full(len(range(0, t.n_parts, 5)), 3, np.int32),
          np.ones(len(range(0, t.n_parts, 5)), np.uint8))
    opts = [{}, dict(has_part_weights=1, weight_overrides=wo), {}]
    full = dict(schedule=list(COUNTS), audit={}, exposure=dict(series_cap=8), span=True, max_concurrent=3)
    return dict(plain=lambda: ctx.plan_chains(t, chains, False, max_concurrent=3),
                exposure=lambda: ctx.plan_chains(t, chains, False, **full),
                exposure_weights=lambda: ctx.plan_chains(t, chains, False, opts=opts, **full))


def test_old_chain_entry_points_launch_as_before(ctx):
    for name, f in parent_launch_arms(ctx).items():
        n, _ = _launches(ctx, f)
        assert n == PARENT_LAUNCHES[name], (name, n)
