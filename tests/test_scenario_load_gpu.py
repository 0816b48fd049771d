"""blance_plan_scenarios_load on the device: every load[i * nc + k] equals blance_moves_load on the handle of scenario
i's rebalance at count k with scenario i's own partition weights (weight overrides included; the vectorised oracle
where a scenario's weights are negative, which the handle refuses), for every wave size; node_end equals the
scenario's state_node_load when nothing is stuck; plans, schedules, audits and exposures equal
blance_plan_scenarios_exposure's; the exposure's launch count is unchanged by an earlier load.  Needs an H100; run
with -m gpu."""
import numpy as np
import pytest

import load_oracle as LO
import scenario_exposure_ref as REF
from test_scenario_audit_gpu import flat
from test_scenario_exposure_gpu import same_exposures, same_schedules
from test_scenario_options_gpu import random_base as random_options_base, random_scenarios as random_option_scenarios
from test_scenarios_gpu import _fresh_then_rebalance, _node_failures, _same_results, random_base, random_scenarios

from blance_b200 import tables

pytestmark = pytest.mark.gpu
COUNTS = (1, 3)


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def handle_load(ctx, t, next_rows, favor, count):
    """blance_moves_load on the handle of scenario tables t's rebalance (begMap partitions), with its weights."""
    member, beg, end = REF.begmap_rows(t, next_rows)
    w = (np.where(np.asarray(t.part_has_weight) != 0, t.part_weight, 1) if t.has_part_weights else np.ones(t.n_parts)).astype(np.int64)[member]
    h, total = ctx.moves_create(t.state_slot_off, beg, end, favor, t.n_node_ids)
    ro, so, _ = ctx.moves_schedule(h, count, (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8))
    if (w >= 0).all():
        got = ctx.moves_load(h, w)
    else:
        off, node, state, kind = ctx.moves_fetch(h, total)
        got = LO.vectorised(t.state_slot_off, beg, off, node, state, kind, ro, so, t.n_node_ids, w)
    ctx.moves_free(h)
    return got


def same_loads(a, b, what):
    for x, y in zip(a.loads, b.loads):
        LO.assert_equal(x, y, what)


def check(ctx, base, scs, opts=None, waves=(1, 3, 0), favors=(False, True), audit=None, exposure=None):
    for favor in favors:
        first = None
        for mc in waves:
            res = ctx.plan_scenarios(base, scs, favor, max_concurrent=mc, want_rows=range(len(scs)), opts=opts,
                                     schedule=list(COUNTS), audit=audit, exposure=exposure, load=True)
            if first is not None:
                for r, q in zip(res, first):
                    same_loads(r, q, (favor, mc))
                continue
            first = res
            plain = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), opts=opts, schedule=list(COUNTS), audit=audit,
                                       exposure=exposure)
            _same_results(res, plain)
            for i, (r, q) in enumerate(zip(res, plain)):
                same_schedules(r, q)
                if audit is not None:
                    assert flat(r.audit) == flat(q.audit), i
                if exposure is not None:
                    same_exposures(r, q, (favor, i))
                t = tables.scenario_tables(base, scs[i], None if opts is None else opts[i])
                for k, c in enumerate(COUNTS):
                    got = r.loads[k]
                    assert got["rounds"] == r.schedules[k].rounds
                    LO.assert_equal(got, handle_load(ctx, t, r.next_rows, favor, c), (favor, i, c))
                    if r.schedules[k].stuck_parts == 0:
                        assert np.array_equal(got["node_end"][:base.n_states], r.state_node_load), (favor, i, c)
    return first


def test_random_bases(ctx):
    for seed in (2, 9):
        t, rng = random_base(seed)
        check(ctx, t, random_scenarios(t, rng, 4))


def test_scenario_weight_overrides(ctx):
    for seed in (3, 11):
        t, _ = random_options_base(seed)
        scs, opts = random_option_scenarios(t, np.random.default_rng(seed), 4)
        check(ctx, t, scs, opts=opts, waves=(1, 0))


def test_with_audit_and_exposure(ctx):
    t, rng = random_base(23)
    check(ctx, t, random_scenarios(t, rng, 3), waves=(2,), favors=(False,), audit=dict(n2n=True), exposure=dict(series_cap=8))


def test_cfg2_node_failures(ctx):
    t = _fresh_then_rebalance(ctx, 2)
    check(ctx, t, _node_failures(t, [[q] for q in range(6)]), waves=(4, 0), favors=(False,))


def test_exposure_launches_unchanged_by_a_load(ctx):
    t, rng = random_base(5)
    scs = random_scenarios(t, rng, 3)

    def launches(**kw):
        n0 = ctx.kernel_launches()
        ctx.plan_scenarios(t, scs, False, max_concurrent=3, schedule=[1, 2], **kw)
        return ctx.kernel_launches() - n0
    before = launches(exposure={}), launches(audit={}), launches()
    launches(load=True)
    assert (launches(exposure={}), launches(audit={}), launches()) == before
