"""blance_map_audit / blance_plan_audit on the device equal the string-map oracle (tests/audit_oracle.py) on random
instances under every option combination, on the synthetic configurations before and after their plans, and a numpy
recomputation on the headline map.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import audit_util as U
from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def check(ctx, inst, what):
    t, rows, shape, names = inst["t"], inst["rows"], inst["shape"], inst["names"]
    for with_rules in (False, True):
        if with_rules:
            U.set_hierarchy(t, inst["parents"], inst["rules"], names)
        for with_forest in (False, True):
            dparents = inst["parents"] if with_forest else None
            arr, vnames = U.forest(t, dparents, names) if with_forest else (None, names)
            e = U.expected(t, U.oracle_of(t, rows, shape, names, inst["parents"], inst["rules"], dparents), names, vnames)
            for n2n in (False, True):
                got = ctx.map_audit(t, rows, shape, n2n=n2n, domain_parent=arr)
                U.assert_audit(got, e, n2n, (what, with_rules, with_forest, n2n))
    return e


@pytest.mark.parametrize("chunk", range(4))
def test_random_instances_equal_the_oracle(ctx, chunk):
    seen_miss = seen_short = 0
    for seed in range(chunk * 6, (chunk + 1) * 6):
        e = check(ctx, U.random_instance(seed), seed)
        seen_miss += e["rule_miss_parts"]
        seen_short += e["short_parts"]
    assert seen_miss > 0 and seen_short > 0


@pytest.mark.parametrize("N,P", [(300, 500), (130, 3000), (33, 6000)])
def test_wide_hierarchies_and_many_partitions(ctx, N, P):
    inst = U.random_instance(1000 + N, N=N, P=P)
    check(ctx, inst, N)
    assert inst["t"].hier_words > 1


def test_domain_tables_beyond_shared_memory(ctx):
    """More than 3 x 44 KB / 4 vertices: the per-vertex counts go to global memory."""
    inst = U.random_instance(77, N=40, P=300)
    t, names = inst["t"], inst["names"]
    dp = dict(inst["parents"])
    dp.update({"pad%05d" % i: "root" for i in range(12000)})
    arr, vnames = U.forest(t, dp, names)
    e = U.expected(t, U.oracle_of(t, inst["rows"], inst["shape"], names, dparents=dp), names, vnames)
    U.assert_audit(ctx.map_audit(t, inst["rows"], inst["shape"], n2n=True, domain_parent=arr), e, True)


def _synth_names(t):
    return ["n%04d" % i for i in range(t.n_nodes)]


def _synth_oracle(cfg, t, rows, shape):
    """cfg's map through the oracle, with synth's state order (priority = index) and its regular tree."""
    c = synth.CONFIGS[cfg]
    names = _synth_names(t)
    parents = synth.node_hierarchy_dict(t.n_nodes, c["levels"])
    rules = {"s%d" % s: list(r) for s, r in c["rules"].items()}
    arr, vnames = U.forest(t, parents, names)
    return U.expected(t, U.oracle_of(t, rows, shape, names, parents, rules, parents), names, vnames), arr


@pytest.mark.parametrize("cfg,P", [(2, None), (3, 4096)])
def test_synthetic_configurations_before_and_after_their_plans(ctx, cfg, P):
    size = {} if P is None else dict(P=P)
    fresh = synth.make_fresh(cfg, **size)
    r0 = ctx.plan_next_map(fresh)
    t = synth.make_rebalance(cfg, r0.next_rows, **size)
    e, arr = _synth_oracle(cfg, t, t.prev_rows, t.prev_shape)
    U.assert_audit(ctx.map_audit(t, t.prev_rows, t.prev_shape, n2n=True, domain_parent=arr), e, True, "before")
    # the resident plan: before the run it holds partitionsToAssign, after it the result
    plan = ctx.upload(t)
    U.assert_audit(ctx.plan_audit(plan, t, n2n=True, domain_parent=arr), e, True, "uploaded")
    ctx.run(plan)
    res = ctx.fetch(plan, tables.PlanResult(t))
    e2, _ = _synth_oracle(cfg, t, res.next_rows, res.next_shape)
    U.assert_audit(ctx.plan_audit(plan, t, n2n=True, domain_parent=arr), e2, True, "resident")
    U.assert_audit(ctx.map_audit(t, res.next_rows, res.next_shape, n2n=True, domain_parent=arr), e2, True, "fetched")
    ctx.free(plan)


def test_headline_map_against_numpy(ctx):
    """cfg 4's 1M x 1024 previous map, nodes only, the failover matrix requested."""
    t = synth.make_rebalance(4)
    rows = np.asarray(t.prev_rows)
    got = ctx.map_audit(t, rows, t.prev_shape, n2n=True)
    N = t.n_nodes
    copies = np.bincount(rows.reshape(-1), minlength=N)
    assert np.array_equal(got.dom_copies, copies)
    assert np.array_equal(got.dom_top, np.bincount(rows[:, 0], minlength=N))
    alone = (rows == rows[:, :1]).all(axis=1)
    assert np.array_equal(got.dom_all, np.bincount(rows[alone, 0], minlength=N))
    n2n = np.zeros((N, N), np.int64)
    for c in range(1, rows.shape[1]):
        sel = rows[:, c] != rows[:, 0]
        np.add.at(n2n, (rows[sel, 0], rows[sel, c]), 1)
    assert np.array_equal(got.n2n, n2n)
    a, b = np.unravel_index(np.argmax(n2n), n2n.shape)                  # the first maximum in (a, b) order
    assert got.n2n_max == (int(n2n.max()), int(a), int(b))
    assert got.short_parts == 0 and got.no_top_parts == 0 and not got.short_slots.any() and not got.over_slots.any()
    assert not got.part_flags.any()
