"""blance_plan_scenarios_audit: audit[i] equals blance_map_audit of scenario i's fetched final map for every wave
size, engine and with or without schedules; plans and schedules are byte-equal to blance_plan_scenarios_schedule;
a rack failure leaves rule misses the planner's warnings never show; the older entry points launch no audit kernel.
Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import audit_util as U
from test_scenarios_gpu import _fresh_then_rebalance, _node_failures, _same_results, random_base, random_scenarios

from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu
FIELDS = ("short_slots", "over_slots", "rule_miss", "rule_tested", "dom_top", "dom_all", "dom_copies", "n2n", "part_flags")


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def final_map(t, r):
    """prevMap with every assigned partition replaced by its next row; a partition in neither map has no lists."""
    assigned, in_prev = (t.part_in_assign != 0)[:, None], (t.part_in_prev != 0)[:, None]
    rows = np.where(assigned, r.next_rows, np.where(in_prev, np.asarray(t.prev_rows).reshape(t.n_parts, -1), -1)).astype(np.int32)
    shape = np.where(assigned, r.next_shape, np.where(in_prev, np.asarray(t.prev_shape).reshape(t.n_parts, -1), 0)).astype(np.uint8)
    return rows, shape


def flat(a):
    return tuple(getattr(a, f).tobytes() for f in FIELDS if getattr(a, f) is not None) + \
        (a.short_parts, a.rule_miss_parts, a.no_top_parts, a.n2n_max)


def check(ctx, base, scs, opts=None, domain_parent=None, schedules=((1, 3), None), waves=(1, 3, 0), engines=(0, 1, 2)):
    audit = dict(n2n=True, domain_parent=domain_parent)
    first = None
    for engine in engines:
        base.engine = engine
        for mc in waves if engine == 0 else (0,):
            for schedule in schedules:
                res = ctx.plan_scenarios(base, scs, False, max_concurrent=mc, want_rows=range(len(scs)), opts=opts,
                                         schedule=None if schedule is None else list(schedule), audit=audit)
                got = [flat(r.audit) for r in res]
                if first is None:
                    first = got
                    plain = ctx.plan_scenarios(base, scs, False, want_rows=range(len(scs)), opts=opts, schedule=list(schedules[0]))
                    _same_results(res, plain)
                    for r, q in zip(res, plain):
                        for a, b in zip(r.schedules, q.schedules):
                            assert (a.rounds, a.moves_done, a.stuck_parts, a.max_batch) == (b.rounds, b.moves_done, b.stuck_parts, b.max_batch)
                            for f in ("node_rounds", "node_last_round", "part_done_round"):
                                assert np.array_equal(getattr(a, f), getattr(b, f))
                    for i, (sc, r) in enumerate(zip(scs, res)):
                        t = tables.scenario_tables(base, sc, None if opts is None else opts[i])
                        rows, shape = final_map(t, r)
                        assert flat(ctx.map_audit(t, rows, shape, n2n=True, domain_parent=domain_parent)) == got[i], i
                else:
                    assert got == first, (engine, mc, schedule)
    base.engine = 0
    return res


def _forest(t, cfg):
    return U.forest(t, synth.node_hierarchy_dict(t.n_nodes, synth.CONFIGS[cfg]["levels"]), ["n%04d" % i for i in range(t.n_nodes)])[0]


def test_cfg2_rack_and_node_failures(ctx):
    t = _fresh_then_rebalance(ctx, 2)
    scs = _node_failures(t, [range(r * 8, r * 8 + 8) for r in range(3)] + [[5], [9, 17], range(8, 64)])
    res = check(ctx, t, scs, domain_parent=_forest(t, 2))
    # the case the audit exists for: every rack but one is gone, each replica falls back into its primary's rack
    # (plan.go:214-220) and no warning says so
    assert res[-1].warn_parts == 0 and res[-1].audit.rule_miss_parts == t.n_parts


def test_cfg3_reduced_rack_failures(ctx):
    t = _fresh_then_rebalance(ctx, 3, P=4096)
    scs = _node_failures(t, [range(0, 8), range(64, 72), [3]])
    check(ctx, t, scs, domain_parent=_forest(t, 3), waves=(1, 0), engines=(0, 1))


def test_random_bases_with_options(ctx):
    for seed in (2, 9, 23):
        t, rng = random_base(seed)
        scs = random_scenarios(t, rng, 4)
        check(ctx, t, scs, schedules=((2,), None), engines=(0,))
    t, rng = random_base(41)
    w = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
    opts = [{}, dict(state_constraints=np.asarray(w.state_constraints, np.int32) + 1), {}]
    check(ctx, w, random_scenarios(w, rng, 3), opts=opts, schedules=((2,), None), engines=(0,))


def test_audit_without_a_schedule_equals_scenarios_ex(ctx):
    t, rng = random_base(5)
    scs = random_scenarios(t, rng, 3)
    res = ctx.plan_scenarios(t, scs, False, want_rows=range(3), audit={})
    _same_results(res, ctx.plan_scenarios(t, scs, False, want_rows=range(3), opts=[{} for _ in scs]))
    assert all(r.schedules is None and r.audit.n2n_max == (-1, -1, -1) for r in res)


def test_older_entry_points_launch_no_audit_kernel(ctx):
    t, rng = random_base(5)
    scs = random_scenarios(t, rng, 3)

    def launches(**kw):
        ctx.plan_scenarios(t, scs, False, max_concurrent=3, **kw)
        n0 = ctx.kernel_launches()
        ctx.plan_scenarios(t, scs, False, max_concurrent=3, **kw)
        return ctx.kernel_launches() - n0
    plain, ex, sched = launches(), launches(opts=[{} for _ in scs]), launches(schedule=[1])
    # one wave: k_map_audit, k_map_audit_rules when the base has rules, k_audit_n2n_max with the matrix
    rules = 1 if t.has_hier_rules and t.n_rules else 0
    assert launches(audit={}) == plain + 1 + rules
    assert launches(audit=dict(n2n=True)) == plain + 2 + rules
    assert launches(schedule=[1], audit={}) == sched + 1 + rules
    assert (launches(), launches(opts=[{} for _ in scs]), launches(schedule=[1])) == (plain, ex, sched)
