"""blance_plan_chain_branches on the device: what-if branches off the stages of a chain.  Every branch output equals
blance_plan_chains_ex on the branch's equivalent chain (its trunk chain's stages up to the fork, then the branch's)
byte for byte, the trunk's outputs equal blance_plan_chains_ex without branches, and no branches at all is that call
with as many kernel launches; none of it depends on the wave size, the engine or the context.  Needs an H100; run
with -m gpu."""
import numpy as np
import pytest

from test_chain_analysis_gpu import summaries
from test_chain_options_gpu import staged_options
from test_chains_gpu import random_chains
from test_exposure_oracle import random_forest
from test_scenario_audit_gpu import flat
from test_scenario_options_gpu import random_base
from test_scenarios_gpu import _same_results
import exposure_oracle as EO

from blance_b200 import tables

pytestmark = pytest.mark.gpu
COUNTS = (1, 3)
BIG = 1 << 15


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def analysis_kw(parent, T, n):
    return dict(want_rows=[(i, t) for i in range(n) for t in range(T)], schedule=list(COUNTS), audit=dict(n2n=True, domain_parent=parent),
                exposure=dict(series_cap=BIG, domain_parent=parent))


def same_stage(x, y, what):
    _same_results([x], [y])
    for s, q in zip(x.schedules, y.schedules):
        for f, v in summaries(s).items():
            assert np.array_equal(v, summaries(q)[f]), (what, f)
    assert flat(x.audit) == flat(y.audit), what
    assert len(x.exposures) == len(y.exposures) == len(COUNTS), what
    for e, g in zip(x.exposures, y.exposures):
        EO.assert_equal(e, g, what)


def same_net(a, b, what):
    assert np.array_equal(a.node_ops, b.node_ops), what
    assert (a.ops_total, a.parts_moved) == (b.ops_total, b.parts_moved), what
    for s, q in zip(a.schedules, b.schedules):
        for f, v in summaries(s).items():
            assert np.array_equal(v, summaries(q)[f]), (what, "net", f)
    for e, g in zip(a.exposures, b.exposures):
        EO.assert_equal(e, g, (what, "net"))


def random_branches(t, rng, chains, sopts, per_point, TB):
    """per_point branches of TB stages at every (chain, after_stage) fork point, after_stage -1 included: random node
    changes (random_chains) with the option patterns of staged_options, which raise a constraint, change stickiness,
    override weights with presence switched both ways, and switch hierarchy rules on."""
    n, T = len(chains), len(chains[0])
    out = []
    for c in range(n):
        for a in range(-1, T):
            stages = random_chains(t, rng, per_point, TB)
            bo = staged_options(t, rng, per_point, TB, kind=int(rng.integers(5)))
            for k in range(per_point):
                out.append(dict(chain=c, after_stage=a, stages=stages[k], stage_opts=bo[k] if rng.random() < 0.8 else None,
                                want_rows=True))
    return out


def check_branches(ctx, t, chains, sopts, branches, favor, parent, **kw):
    """One call with branches against blance_plan_chains_ex without them (the trunk) and on every equivalent chain."""
    n, T = len(chains), len(chains[0])
    args = analysis_kw(parent, T, n)
    args.update(kw)
    res, nets, bres, bnets = ctx.plan_chains(t, chains, favor, stage_opts=sopts, branches=branches, **args)
    tres, tnets = ctx.plan_chains(t, chains, favor, stage_opts=sopts, **args)
    for i in range(n):
        for s in range(T):
            same_stage(res[i][s], tres[i][s], ("trunk", i, s))
        same_net(nets[i], tnets[i], ("trunk", i))
    for b, br in enumerate(branches):
        c, a = br["chain"], br["after_stage"]
        TB = len(br["stages"])
        eq = chains[c][:a + 1] + br["stages"]
        eo = sopts[c][:a + 1] + (br["stage_opts"] if br["stage_opts"] is not None else [{}] * TB)
        eargs = analysis_kw(parent, len(eq), 1)
        eargs.update(kw)
        er, en = ctx.plan_chains(t, [eq], favor, stage_opts=[eo], **eargs)
        for u in range(TB):
            same_stage(bres[b][u], er[0][a + 1 + u], ("branch", b, u))
        same_net(bnets[b], en[0], ("branch", b))
    return res, nets, bres, bnets


def _launches(ctx, f):
    f()
    n0 = ctx.kernel_launches()
    r = f()
    return ctx.kernel_launches() - n0, r


def test_no_branches_is_chains_ex(ctx):
    t, rng = random_base(17)
    T = 3
    chains = random_chains(t, rng, 4, T)
    sopts = staged_options(t, rng, 4, T)
    parent = random_forest(rng, t.n_node_ids, 3)
    kw = analysis_kw(parent, T, 4)
    la, a = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=sopts, **kw))
    lb, b = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=sopts, branches=[], **kw))
    for i in range(4):
        for s in range(T):
            same_stage(a[0][i][s], b[0][i][s], (i, s))
        same_net(a[1][i], b[1][i], i)
    assert b[2] == [] and b[3] == []
    assert la == lb, (la, lb)
    # without a schedule
    lp, p = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=sopts, want_rows=kw["want_rows"]))
    lq, q = _launches(ctx, lambda: ctx.plan_chains(t, chains, True, stage_opts=sopts, want_rows=kw["want_rows"], branches=[]))
    for i in range(4):
        _same_results(p[0][i], q[0][i])
    assert lp == lq, (lp, lq)


@pytest.mark.parametrize("seed,TB", [(3, 1), (8, 2), (21, 1), (30, 2), (4, 1), (13, 2)])
def test_random_branches_equal_equivalent_chains(ctx, seed, TB):
    t, rng = random_base(seed)
    T = 2 + seed % 3                   # T = 2, 4, 2, 2, 3, 3: after_stage takes -1, 0, middle stages and T - 1
    chains = random_chains(t, rng, 3, T)
    sopts = staged_options(t, rng, 3, T)
    parent = random_forest(rng, t.n_node_ids, 3)
    branches = random_branches(t, rng, chains, sopts, 1, TB)
    check_branches(ctx, t, chains, sopts, branches, bool(seed % 2), parent)


def test_independent_of_wave_size_engine_and_context(ctx, monkeypatch):
    t, rng = random_base(12)
    T = 3
    chains = random_chains(t, rng, 3, T)
    sopts = staged_options(t, rng, 3, T)
    parent = random_forest(rng, t.n_node_ids, 3)
    branches = random_branches(t, rng, chains, sopts, 2, 1)
    args = analysis_kw(parent, T, 3)
    first = ctx.plan_chains(t, chains, False, stage_opts=sopts, branches=branches, **args)

    def same(other, what):
        for i in range(3):
            for s in range(T):
                same_stage(first[0][i][s], other[0][i][s], (what, i, s))
            same_net(first[1][i], other[1][i], (what, i))
        for b in range(len(branches)):
            same_stage(first[2][b][0], other[2][b][0], (what, "branch", b))
            same_net(first[3][b], other[3][b], (what, "branch", b))

    for mc in (1, 2, 0):
        same(ctx.plan_chains(t, chains, False, stage_opts=sopts, branches=branches, max_concurrent=mc, **args), ("mc", mc))
    for env in ("BLANCE_NO_SPEC", "BLANCE_NO_SEQ"):
        monkeypatch.setenv(env, "1")
        same(ctx.plan_chains(t, chains, False, stage_opts=sopts, branches=branches, **args), env)
        monkeypatch.delenv(env)
    multi = tables.Context(device_ids=[0])
    try:
        same(multi.plan_chains(t, chains, False, stage_opts=sopts, branches=branches, **args), "multi")
    finally:
        multi.close()


def test_one_trunk_chain_and_more_branches_than_a_wave(ctx):
    """One trunk chain (which would otherwise plan on the base upload itself) and five branches at one stage, planned
    two at a time."""
    t, rng = random_base(5)
    T = 3
    chains = random_chains(t, rng, 1, T)
    sopts = staged_options(t, rng, 1, T, kind=2)
    parent = random_forest(rng, t.n_node_ids, 2)
    stages = random_chains(t, rng, 5, 1)
    branches = [dict(chain=0, after_stage=1, stages=stages[k], stage_opts=None, want_rows=True) for k in range(5)]
    branches.append(dict(chain=0, after_stage=-1, stages=stages[0], stage_opts=None, want_rows=True))
    check_branches(ctx, t, chains, sopts, branches, True, parent, max_concurrent=2)


def test_without_schedule(ctx):
    t, rng = random_base(9)
    T = 2
    chains = random_chains(t, rng, 2, T)
    sopts = staged_options(t, rng, 2, T)
    branches = random_branches(t, rng, chains, sopts, 1, 2)
    want = [(i, s) for i in range(2) for s in range(T)]
    res, nets, bres, bnets = ctx.plan_chains(t, chains, False, stage_opts=sopts, branches=branches, want_rows=want)
    for b, br in enumerate(branches):
        c, a = br["chain"], br["after_stage"]
        eq = chains[c][:a + 1] + br["stages"]
        eo = sopts[c][:a + 1] + (br["stage_opts"] if br["stage_opts"] is not None else [{}] * 2)
        er, en = ctx.plan_chains(t, [eq], False, stage_opts=[eo], want_rows=[(0, s) for s in range(len(eq))])
        _same_results(bres[b], er[0][a + 1:])
        assert np.array_equal(bnets[b].node_ops, en[0].node_ops) and bnets[b].ops_total == en[0].ops_total


# ---- the string face against the literal Go loop on the equivalent chains -----------------------------------------

def _default_members(universe, stage):
    """The members a branch stage without nodesAll starts from after trunk stage `stage` (nodesAll_t, remove, add, nw):
    its nodesAll minus its removals, in universe order."""
    nodes_all, rm = stage[0], set(stage[1] or [])
    return [n for n in universe if n in nodes_all and n not in rm]


@pytest.mark.parametrize("chunk", range(2))
def test_string_face_branches_equal_literal_loop(chunk):
    import random

    import chain_stage_util as CS
    from randgen import random_instance
    from test_chain_options_gpu import _string_stages
    from test_chains import make_chain
    from test_scenario_options import options_of
    from test_scenarios import removal_allowed
    import blance_b200

    checked = 0
    for seed in range(chunk * 15, (chunk + 1) * 15):
        kw = random_instance(seed)
        if not removal_allowed(kw) and kw["nodes_to_remove"]:
            continue
        stages = make_chain(kw, seed)
        if not removal_allowed(kw):
            stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
        keys = CS.make_stage_options(kw, seed, len(stages))
        universe = kw["nodes_all"]
        rnd = random.Random(seed)
        branches, equivalent = [], []
        for a in range(-1, len(stages)):
            members = list(universe) if a < 0 else _default_members(universe, stages[a])
            absent = [n for n in universe if n not in members]
            if absent and rnd.random() < 0.4:
                rm, add = [], [rnd.choice(absent)]
            elif len(members) > 1 and (a >= 0 or removal_allowed(kw)):
                rm, add = [rnd.choice(members)], []
            else:
                rm, add = [], None
            own = {} if rnd.random() < 0.5 else CS.make_stage_options(kw, seed + 1, 1)[0]
            branches.append({"chain": 0, "afterStage": a, "wantMaps": True,
                             "stages": [dict(own, nodesToRemove=rm, nodesToAdd=add)]})   # nodesAll: the default
            nodes_all = [n for n in universe if n in members or n in (add or [])]
            equivalent.append((stages[:a + 1] + [(nodes_all, rm, add, "inherit")], keys[:a + 1] + [own]))
        prev, assign = kw["prev_map"], kw["partitions_to_assign"]
        chain = {"stages": _string_stages(stages, keys)}
        res, bres = blance_b200.PlanNextMapChains(prev, prev if assign is None else assign, universe, kw["model"], options_of(kw),
                                                  [chain], seed % 2 == 1, wantMaps=[0], branches=branches)
        plain = blance_b200.PlanNextMapChains(prev, prev if assign is None else assign, universe, kw["model"], options_of(kw),
                                              [chain], seed % 2 == 1, wantMaps=[0])
        for t in range(len(stages)):
            for f in ("next_map", "warnings", "ops_total", "node_ops", "iterations"):
                assert res[0]["stages"][t].get(f) == plain[0]["stages"][t].get(f), (seed, t, f)
        for b, (eq_stages, eq_keys) in enumerate(equivalent):
            lit = CS.literal_chain_staged(kw, eq_stages, eq_keys)[-1]
            r = bres[b]["stages"][0]
            assert r["iterations"] == lit["iterations"], (seed, b)
            assert r["next_map"] == (lit["next_map"] if r["iterations"] > 0 else {}), (seed, b)
            assert r["warnings"] == (lit["warnings"] if r["iterations"] > 0 else {}), (seed, b)
        checked += 1
    assert checked > 5
