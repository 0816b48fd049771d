"""blance_plan_scenarios_exposure on the device: every expo[i * nc + k] equals, field for field, blance_moves_exposure
on the handle of scenario i's rebalance at count k and the CPU reference (tests/scenario_exposure_ref.py), for every
wave size, engine and a multi-device context, with and without an audit, for both favor_min_nodes; plans, schedules
and audits are byte-equal to blance_plan_scenarios_audit / _schedule; the series is cut at series_cap; the older
entry points launch no exposure kernel.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import exposure_oracle as EO
import scenario_exposure_ref as REF
from test_scenario_audit_gpu import _forest, flat
from test_scenarios_gpu import _fresh_then_rebalance, _node_failures, _same_results, random_base, random_scenarios

from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu
COUNTS = (1, 3)
BIG = 1 << 15                                   # a series cap above any R here (host buffers are [6][cap] per pair)


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def handle_exposure(ctx, t, next_rows, favor, count, parent):
    """blance_moves_exposure on the handle of the scenario's rebalance (begMap partitions), scattered to [n_parts]."""
    member, beg, end = REF.begmap_rows(t, next_rows)
    h, _ = ctx.moves_create(t.state_slot_off, beg, end, favor, t.n_node_ids)
    ctx.moves_schedule(h, count, (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8))
    got = ctx.moves_exposure(h, np.asarray(t.state_constraints, np.int32), t.top_state, parent)
    ctx.moves_free(h)
    for k, fill, dt in REF.PART_FILL:
        full = np.full(t.n_parts, fill, dt)
        full[member] = got[k]
        got[k] = full
    return got


def same_schedules(a, b):
    for x, y in zip(a.schedules, b.schedules):
        assert (x.rounds, x.moves_done, x.stuck_parts, x.max_batch) == (y.rounds, y.moves_done, y.stuck_parts, y.max_batch)
        for f in ("node_rounds", "node_last_round", "part_done_round"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), f


def same_exposures(a, b, what):
    for x, y in zip(a.exposures, b.exposures):
        EO.assert_equal(x, y, what)


def check(ctx, base, scs, opts=None, parent=None, waves=(1, 3, 0), engines=(0, 1, 2), audits=(None, dict(n2n=True)), favors=(False, True),
          reference=True):
    expo = dict(domain_parent=parent, series_cap=BIG)
    for favor in favors:
        first = None
        for audit in audits:
            for engine in engines:
                base.engine = engine
                for mc in waves if engine == 0 else (0,):
                    res = ctx.plan_scenarios(base, scs, favor, max_concurrent=mc, want_rows=range(len(scs)), opts=opts,
                                             schedule=list(COUNTS), audit=audit, exposure=expo)
                    if first is not None:
                        for r, q in zip(res, first):
                            same_exposures(r, q, (favor, audit, engine, mc))
                        continue
                    first = res
                    plain = ctx.plan_scenarios(base, scs, favor, want_rows=range(len(scs)), opts=opts, schedule=list(COUNTS), audit=audit)
                    _same_results(res, plain)
                    for i, (r, q) in enumerate(zip(res, plain)):
                        same_schedules(r, q)
                        if audit is not None:
                            assert flat(r.audit) == flat(q.audit), i
                        t = tables.scenario_tables(base, scs[i], None if opts is None else opts[i])
                        for k, c in enumerate(COUNTS):
                            got = r.exposures[k]
                            assert got["rounds"] == r.schedules[k].rounds
                            EO.assert_equal(got, handle_exposure(ctx, t, r.next_rows, favor, c, parent), (favor, i, c, "handle"))
                            if reference:
                                want, _ = REF.scenario_exposure(t, r.next_rows, favor, c, domain_parent=parent)
                                EO.assert_equal(got, want, (favor, i, c, "reference"))
    base.engine = 0
    return first


def _with_neither(t, rng):
    P = t.n_parts
    t.part_in_assign[:] = (rng.random(P) < 0.7).astype(np.uint8)
    gone = rng.random(P) < 0.1
    t.part_in_prev[gone] = 0
    t.part_in_assign[gone] = 0
    t.prev_rows.reshape(P, -1)[gone] = -1
    t.prev_shape.reshape(P, -1)[gone] = 0
    return t, gone


def test_random_bases_with_options(ctx):
    for seed in (2, 9, 23):
        t, rng = random_base(seed)
        check(ctx, t, random_scenarios(t, rng, 4), waves=(1, 3, 0), engines=(0,))
    t, rng = random_base(41)
    w = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
    opts = [{}, dict(state_constraints=np.asarray(w.state_constraints, np.int32) + 1), {}]
    res = check(ctx, w, random_scenarios(w, rng, 3), opts=opts, engines=(0, 1, 2))
    # raised constraints: the partitions are SHORT at t = 0 and the new copies are counted as they land
    assert res[1].exposures[0]["series"][EO.METRICS.index("SHORT"), 0] > 0


def test_partitions_in_neither_map(ctx):
    t, rng = random_base(12)
    t, gone = _with_neither(t, rng)
    scs = random_scenarios(t, rng, 3)
    for sc in scs:                               # plan.go:544: no removal with partitions absent from prevMap
        sc["node_removed"][:] = 0
    res = check(ctx, t, scs, waves=(0,), engines=(0,))
    for r in res:
        for e in r.exposures:
            assert (e["part_min_copies"][gone] == -1).all()
            assert not e["part_no_top"][gone].any() and not e["part_flags"][gone].any()


def test_cfg2_rack_forest(ctx):
    t = _fresh_then_rebalance(ctx, 2)
    scs = _node_failures(t, [range(0, 8), [5], [9, 17]])
    check(ctx, t, scs, parent=_forest(t, 2), waves=(1, 0), engines=(0, 2))


def test_cfg3_reduced(ctx):
    t = _fresh_then_rebalance(ctx, 3, P=4096)
    scs = _node_failures(t, [range(0, 8), [3]])
    check(ctx, t, scs, parent=_forest(t, 3), waves=(0,), engines=(0,), audits=(None,))


def test_cfg4_reduced(ctx):
    t = synth.make_rebalance(4, P=16384)
    scs = _node_failures(t, [[j] for j in range(3)])
    check(ctx, t, scs, waves=(0,), engines=(0,), audits=(None,), reference=False)


def test_multi_device_context(ctx):
    t, rng = random_base(7)
    scs = random_scenarios(t, rng, 5)
    expo = dict(series_cap=BIG)
    first = ctx.plan_scenarios(t, scs, True, want_rows=range(5), schedule=list(COUNTS), exposure=expo)
    multi = tables.Context(device_ids=[0])
    try:
        again = multi.plan_scenarios(t, scs, True, want_rows=range(5), schedule=list(COUNTS), exposure=expo)
    finally:
        multi.close()
    _same_results(first, again)
    for a, b in zip(first, again):
        same_exposures(a, b, "multi")


def test_series_cap(ctx):
    t, rng = random_base(9)
    scs = random_scenarios(t, rng, 3)
    full = ctx.plan_scenarios(t, scs, False, schedule=list(COUNTS), exposure=dict(series_cap=BIG))
    R = max(e["rounds"] for r in full for e in r.exposures)
    assert R > 1
    for cap in (1, R, R + 1, R + 7, 0):
        cut = ctx.plan_scenarios(t, scs, False, schedule=list(COUNTS), exposure=dict(series_cap=cap))
        for a, b in zip(full, cut):
            for x, y in zip(a.exposures, b.exposures):
                n = min(x["rounds"] + 1, cap)
                assert y["series"].shape == (6, n) and np.array_equal(y["series"], x["series"][:, :n])
                for k in ("rounds", "peak", "peak_round", "area", "dom_peak", "dom_peak_round", "part_min_copies", "part_no_top", "part_flags"):
                    assert np.array_equal(x[k], y[k]), (cap, k)
    # dom=False: no fault-domain work; parts=False: no per-partition arrays; everything else the same
    for kw, gone in ((dict(dom=False), ("dom_peak", "dom_peak_round")),
                     (dict(parts=False), ("part_min_copies", "part_no_top", "part_flags"))):
        less = ctx.plan_scenarios(t, scs, False, schedule=list(COUNTS), exposure=dict(series_cap=BIG, **kw))
        for a, b in zip(full, less):
            for x, y in zip(a.exposures, b.exposures):
                assert not set(gone) & set(y)
                for k in set(y) - {"kernel_ms"}:
                    assert np.array_equal(x[k], y[k]), (kw, k)


# kernels launched by the second of two identical calls on random_base(5) with 3 scenarios at max_concurrent = 3,
# counted with the build before blance_plan_scenarios_exposure existed
PARENT_LAUNCHES = dict(plain=73, ex=73, sched1=461, sched12=461, audit1=462)


def test_launches(ctx):
    t, rng = random_base(5)
    scs = random_scenarios(t, rng, 3)

    def launches(**kw):
        ctx.plan_scenarios(t, scs, False, max_concurrent=3, **kw)
        n0 = ctx.kernel_launches()
        ctx.plan_scenarios(t, scs, False, max_concurrent=3, **kw)
        return ctx.kernel_launches() - n0
    plain, ex, sched, aud = launches(), launches(opts=[{} for _ in scs]), launches(schedule=[1]), launches(schedule=[1], audit={})
    sched12 = launches(schedule=[1, 2])
    assert dict(plain=plain, ex=ex, sched1=sched, sched12=sched12, audit1=aud) == PARENT_LAUNCHES
    # one wave: k_expo_walk<0> and k_expo_series; with dom peaks k_expo_dom_init, k_expo_walk<1> and, for the one
    # group of events, k_expo_walk<2> and k_expo_dom_max
    assert launches(schedule=[1], exposure=dict(dom=False)) == sched + 2
    assert launches(schedule=[1], audit={}, exposure=dict(dom=False)) == aud + 2
    assert launches(schedule=[1, 2], exposure=dict(dom=False)) == sched12 + 2
    assert launches(schedule=[1], exposure={}) == sched + 6
    # an exposure leaves nothing behind that changes a later call of an older entry point
    assert dict(plain=launches(), ex=launches(opts=[{} for _ in scs]), sched1=launches(schedule=[1]), sched12=launches(schedule=[1, 2]),
                audit1=launches(schedule=[1], audit={})) == PARENT_LAUNCHES


def _tiny_base(seed, P=12, N=8):
    rng = np.random.default_rng(seed)
    t = tables.PlanTables(N, 2, P, [0, 1], [1, 1], n_node_ids=N)
    rows = np.stack([rng.permutation(N - 2)[:2] for _ in range(P)]).astype(np.int32)
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:] = 2
    t.cur_shape[:] = 2
    t.part_in_prev[:] = 1
    t.max_iters = 3
    return t, rng


def test_more_than_65535_instances_in_one_event_group(ctx):
    """8 200 scenarios x 8 counts = 65 600 (scenario, count) pairs in one wave and one fault-domain event group: the
    emitting walk is split into launches of 65 535 instances, and the events of instance 65 535 + x must not merge with
    those of instance x.  Scenarios on both sides of the split equal the same scenarios planned alone."""
    t, rng = _tiny_base(3)
    counts = list(range(1, 9))
    scs = []
    for j in range(8200):
        rm = np.zeros(t.n_node_ids, np.uint8)
        rm[int(rng.integers(0, t.n_nodes - 2))] = 1
        ad = np.zeros(t.n_node_ids, np.uint8)
        ad[t.n_nodes - 1 - j % 2] = 1
        scs.append(dict(node_removed=rm, node_added=ad, add_is_nil=0))
    expo = dict(series_cap=64)                         # the host buffers are [6][cap] per pair: 65 600 of them
    big = ctx.plan_scenarios(t, scs, False, schedule=counts, exposure=expo)
    sample = [0, 1, 2, 8190, 8191, 8192, 8199]         # instance 65 535 is scenario 8 191, count index 7
    alone = ctx.plan_scenarios(t, [scs[j] for j in sample], False, schedule=counts, exposure=expo)
    moved = 0
    for j, r in zip(sample, alone):
        for a, b in zip(big[j].exposures, r.exposures):
            for k in set(a) - {"kernel_ms"}:
                assert np.array_equal(a[k], b[k]), (j, k)
            moved += int(a["rounds"] > 0)
    assert moved > 0                                   # the sample has rebalances, so it has fault-domain events
