"""The three pass kernels at the extremes of the values that feed the score (plan.go:634-689): partition weights
negative, zero and up to 999 999 999, StateStickiness 0, 2^31 - 1 and negative, node weights from -2^31 to 2^31 - 1
with and without the booster, and node totals just under INT32_MAX (the count bound of include/blance_b200.h).

Every case plans against the array-form CPU oracle on the same tables (rows, shapes, warnings, iterations,
convergence, steps) on the speculative, sequencer and lock-step kernels, and checks which kernel ran: the lock-step
kernel decides no step without a full evaluation (sticky_steps == 0); the sequencer and the speculative kernel do
where rows keep positive stickiness (sticky_steps > 0).  Where no step can be sticky, the speculative kernel's
path counters (BLANCE_SPEC_STATS) show that it ran: steps resolved by its leader or movers.  Each family that
cannot be sticky has a sibling in which most rows keep positive stickiness.  test_value_range.py shows the
literal oracle equal to the array-form one at these values.  Needs an H100; run with `-m gpu`."""
import copy
import random
import re

import numpy as np
import pytest

from oracle_loader import literal
from test_engine_limits_gpu import FAST, LOCK, SEQ, SPEC, assert_kernel, assert_same, cluster, oracle_tables, set_engine
from test_scenario_options_gpu import check_against_oracle
from test_value_range import I32_MAX, wrapping_instance

import blance_b200
from blance_b200 import _host, abi, tables

pytestmark = pytest.mark.gpu

I32_MIN = -2**31
STATS = re.compile(r"\[blance\] inst \d+: steps \d+ accepted (\d+) \| resolved by the leader (\d+) .* movers (\d+) ")


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def spec_ran(err):
    """Sum of (leader resolves + movers) over the BLANCE_SPEC_STATS lines of one call."""
    return sum(int(m.group(2)) + int(m.group(3)) for m in map(STATS.search, err.splitlines()) if m)


def plan_every_kernel(ctx, monkeypatch, capfd, t, sticky, what):
    """Plans t on each kernel against the oracle; `sticky`: most rows keep positive stickiness, so both sticky kernels
    must decide some steps alone."""
    ref = oracle_tables(t)
    monkeypatch.setenv("BLANCE_SPEC_STATS", "1")
    for kernel in (SPEC, SEQ, LOCK):
        set_engine(monkeypatch, t, kernel)
        capfd.readouterr()
        got = ctx.plan_next_map(t)
        err = capfd.readouterr().err
        assert_same(got, ref, (what, kernel))
        if kernel == LOCK or sticky:
            assert_kernel(got, kernel, (what, kernel))
        if kernel == SPEC:
            assert got.sticky_steps > 0 or spec_ran(err) > 0, (what, err[-1000:])
    return ref


# ---- value families -------------------------------------------------------------------------------------------

def weigh(t, mask, w):
    t.part_has_weight[:] = mask
    t.part_weight[:] = np.where(mask, w, 1)


def largest_fitting(t, n_big):
    """The largest weight (at most 999 999 999) that n_big partitions can carry with every other one at weight 1."""
    return int(min(999999999, (I32_MAX - (t.n_parts - n_big) * t.n_slots) // (n_big * t.n_slots)))


def f_neg(frac):
    def f(t, rng):
        weigh(t, rng.random(t.n_parts) < frac, -rng.choice([1, 7, 1000, 100000], t.n_parts))
    return f


def f_zero(frac):
    def f(t, rng):
        weigh(t, rng.random(t.n_parts) < frac, 0)
    return f


def f_huge_few(t, rng):
    n_big = 3
    big = rng.choice(t.n_parts, n_big, replace=False)
    mask = np.ones(t.n_parts, bool)
    weigh(t, mask, 1)
    t.part_weight[big] = largest_fitting(t, n_big)


def f_stick(v, weighted=False):
    def f(t, rng):
        if not weighted:
            weigh(t, np.zeros(t.n_parts, bool), 1)
        t.state_stickiness[:] = v
    return f


def f_nw_mixed(t, rng):
    t.node_weight[:] = np.where(rng.random(t.n_nodes) < 0.5, I32_MAX, 1)


def f_nw_equal(v):
    def f(t, rng):
        t.node_weight[:] = v
    return f


def f_nw_negative(booster, stick):
    """Node weights 0, negative (down to -2^31) and 1-2; stickiness `stick` for state 0 and 5 for the rest, so that
    max(-w, stickiness) (the booster) takes either side."""
    def f(t, rng):
        t.node_weight[:] = rng.choice([I32_MIN, -3, -3, -1, 0, 0, 1, 2], t.n_nodes)
        t.booster_kind = booster
        weigh(t, np.zeros(t.n_parts, bool), 1)
        t.state_stickiness[:] = 5
        t.state_stickiness[0] = stick
    return f


# name: (mutation, most rows keep positive stickiness)
FAMILIES = {
    "neg_weights_quarter": (f_neg(0.25), True),
    "neg_weights_all": (f_neg(1.0), False),
    "zero_weights_half": (f_zero(0.5), True),
    "zero_weights_all": (f_zero(1.0), False),
    "huge_weights_few": (f_huge_few, True),
    "stickiness_0": (f_stick(0), False),
    "stickiness_max": (f_stick(I32_MAX), True),
    "stickiness_negative": (f_stick(-5), False),
    "stickiness_negative_quarter_weighted": (f_stick(-5, weighted=True), True),
    "node_weights_max_mixed": (f_nw_mixed, True),
    "node_weights_equal_huge": (f_nw_equal(I32_MAX), True),
    "node_weights_equal_2_30": (f_nw_equal(2**30), True),
    "node_weights_negative_booster": (f_nw_negative(blance_b200.BOOSTER_CBGT_MAX, 2), True),
    "node_weights_negative_no_booster": (f_nw_negative(blance_b200.BOOSTER_NONE, 2), True),
    "node_weights_negative_booster_stick_negative": (f_nw_negative(blance_b200.BOOSTER_CBGT_MAX, -5), False),
}


def family(name, N, K, seed=0, P=2048):
    t = cluster(N, P, [1, K], n_rm=2, n_add=2, seed=seed)
    FAMILIES[name][0](t, np.random.default_rng(seed + 7))
    return t


@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("N", [96, 1024, 2048])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_value_families_every_kernel(ctx, monkeypatch, capfd, name, N, K):
    plan_every_kernel(ctx, monkeypatch, capfd, family(name, N, K, seed=N + K), FAMILIES[name][1], (name, N, K))


# ---- at the edge of int32 -------------------------------------------------------------------------------------

@pytest.mark.parametrize("extra", [0, 12345])
def test_node_total_just_under_int32_max(ctx, monkeypatch, capfd, extra):
    """One slot per row; three partitions on node 5 carry all but (n_parts - 3) + extra of INT32_MAX, the rest weigh
    1 and `extra` is node 5's count of non-model states: node 5's total starts within n_parts of INT32_MAX and the
    instance sits exactly at the count bound."""
    t = cluster(256, 2048, [1], n_rm=2, n_add=2, seed=11)
    weigh(t, np.ones(t.n_parts, bool), 1)
    t.prev_rows[:3, 0] = 5
    t.cur_rows[:3, 0] = 5
    rest = I32_MAX - (t.n_parts - 3) - extra
    t.part_weight[:3] = [999999999, 999999999, rest - 2 * 999999999]
    t.extra_tot_first[5] = extra
    t.extra_tot_rest[5] = extra
    assert int(np.abs(t.part_weight.astype(np.int64)).sum()) + extra == I32_MAX
    start = int(t.part_weight[t.prev_rows[:, 0] == 5].astype(np.int64).sum()) + extra
    assert I32_MAX - start < t.n_parts
    plan_every_kernel(ctx, monkeypatch, capfd, t, True, ("edge", extra))


def test_string_api_refuses_counts_that_wrap():
    kw = wrapping_instance()
    o = blance_b200.PlanNextMapOptions(PartitionWeights=kw["partition_weights"])
    with pytest.raises(blance_b200.BlanceError, match="exceeds int32"):
        blance_b200.PlanNextMapEx(kw["prev_map"], kw["partitions_to_assign"], kw["nodes_all"], kw["nodes_to_remove"],
                                  kw["nodes_to_add"], kw["model"], o)


# ---- the option space at sticky-kernel sizes (string form) -------------------------------------------------------

def midsize_instance(seed):
    """A string-form instance of 200-3 000 partitions: partitions only in partitionsToAssign, an empty prevMap with
    a filled partitionsToAssign, non-model entries (on unassigned and on assigned partitions), a few nil / absent
    lists, duplicates and nodes outside nodesAll, equal priorities, constraint overrides, hierarchy rules on the
    replica state only, and extreme weights and stickiness within the count bound."""
    rnd = random.Random("value range midsize %d" % seed)
    nodes = ["n%03d" % i for i in range(rnd.choice([24, 64, 200]))]
    P = rnd.randint(200, 3000)
    k = rnd.randint(1, 3)
    model = {"primary": (0, 1), "replica": (0 if rnd.random() < 0.2 else 1, k)}
    names = [str(i) for i in range(P)]

    def row(allow_odd):
        r = rnd.sample(nodes, k + 1)
        nbs = {"primary": r[:1], "replica": r[1:]}
        if allow_odd and rnd.random() < 0.004:
            x = rnd.random()
            if x < 0.25:
                nbs["replica"] = None
            elif x < 0.5:
                del nbs["replica"]
            elif x < 0.75:
                nbs["replica"] = nbs["replica"] + nbs["replica"][:1]
            else:
                nbs["replica"] = nbs["replica"][:-1] + ["ghost%d" % rnd.randint(0, 3)]
        return nbs

    empty_prev = rnd.random() < 0.2
    prev = {} if empty_prev else {n: row(True) for n in names}
    if empty_prev:
        assign = {n: {} for n in names}                         # P = 0 in iteration 1, then P = n
    elif rnd.random() < 0.4:
        assign = None                                           # the same map
    else:
        assign = {n: {s: (None if v is None else list(v)) for s, v in prev[n].items()} for n in names if rnd.random() < 0.8}
        assign.update({"x%d" % i: {} for i in range(rnd.randint(1, 20))})     # only in partitionsToAssign
    if assign is not None and not empty_prev:
        for n in rnd.sample(names, 3):                          # non-model entries: extras, part_in_prev = 3 if assigned
            prev[n] = dict(prev[n], dead=[rnd.choice(nodes)])
    remove = rnd.sample(nodes, rnd.randint(0, 2))
    if empty_prev or (assign is not None and any(n not in prev for n in assign)):
        remove = []                                             # the reference panics otherwise (plan.go:544)
    add = rnd.choice([None, [], rnd.sample(nodes, 2)])
    kw = dict(prev_map=prev, partitions_to_assign=assign, nodes_all=nodes, nodes_to_remove=remove, nodes_to_add=add,
              model=model)
    if rnd.random() < 0.3:
        kw["model_state_constraints"] = {"replica": rnd.randint(1, 3)}
    if rnd.random() < 0.7:
        kw["partition_weights"] = {n: rnd.choice([-10**9, -7, -1, 0, 1, 999999999, 2, 3]) for n in names if rnd.random() < 0.1}
        kw["state_stickiness"] = {s: rnd.choice([-5, 0, 2, 3, I32_MAX]) for s in model if rnd.random() < 0.8}
    if rnd.random() < 0.6:
        kw["node_weights"] = {n: rnd.choice([I32_MIN, -1, 0, 1, 2, 2**30, I32_MAX]) for n in nodes if rnd.random() < 0.5}
        kw["booster"] = rnd.randint(0, 1)
    if rnd.random() < 0.3:
        kw["node_hierarchy"] = {n: "rack%d" % (i // 4) for i, n in enumerate(nodes)}
        kw["hierarchy_rules"] = {"replica": [(1, 0)]}
    while True:
        try:
            return kw, _host.intern_plan(**copy.deepcopy(kw))
        except blance_b200.BlanceError as e:
            if "exceeds int32" not in str(e):
                raise
            w = kw["partition_weights"]
            for n in sorted(w, key=lambda n: -abs(w[n]))[:8]:
                w[n] = rnd.choice((-7, -1, 0, 1))


def test_option_space_at_sticky_kernel_sizes(monkeypatch):
    L = literal()
    n_seeds, sticky = 24, 0
    for seed in range(n_seeds):
        kw, ip = midsize_instance(seed)
        ref = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, ref.out_ptr) == 0
        ran = 0
        for kernel, engine in ((SPEC, 0), (SEQ, 2), (LOCK, 1)):
            if kernel == SPEC:
                monkeypatch.setenv("BLANCE_NO_SEQ", "1")
            else:
                monkeypatch.delenv("BLANCE_NO_SEQ", raising=False)
            ip.set_engine(engine)
            got = _host.plan_out(ip)
            _host.run_plan_cuda(ip, got)
            what = (seed, kernel)
            assert np.array_equal(got.next_rows, ref.next_rows), what
            assert np.array_equal(got.next_shape, ref.next_shape), what
            assert np.array_equal(got.warn, ref.warn), what
            assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps), what
            st = abi.PlanOut.from_address(got.out_ptr).sticky_steps
            if kernel == LOCK:
                assert st == 0, what
            ran += st > 0
        sticky += ran > 0
        if seed % 10 == 0:
            monkeypatch.delenv("BLANCE_NO_SEQ", raising=False)
            lit = L.plan_next_map_ex(**copy.deepcopy(kw))
            r = _host.PlanNextMapEx(**copy.deepcopy(kw))
            assert r["next_map"] == lit["next_map"] and r["warnings"] == lit["warnings"], seed
    assert 2 * sticky > n_seeds, sticky


# ---- batch and scenarios --------------------------------------------------------------------------------------

def test_value_families_in_one_narrow_batch(ctx, monkeypatch, sm_count):
    """More than sm_count / 2 instances (the narrow 4-scout launch of the speculative kernel), every family, K = 1..4
    and the three engines side by side."""
    monkeypatch.delenv("BLANCE_NO_SEQ", raising=False)
    names = list(FAMILIES)
    n = sm_count // 2 + 3
    ts, ran = [], []
    for i in range(n):
        name = names[i % len(names)]
        kernel = (SPEC, SEQ, LOCK)[(i // len(names)) % 3]
        t = family(name, 256, 1 + i % 4, seed=i, P=1024 + 8 * i)
        t.engine = {SPEC: 0, SEQ: 2, LOCK: 1}[kernel]
        ts.append(t)
        ran.append((kernel, FAMILIES[name][1]))
    for i, (g, t) in enumerate(zip(ctx.plan_next_map_batch(ts), ts)):
        assert_same(g, oracle_tables(t), i)
        kernel, sticky = ran[i]
        if kernel == LOCK or sticky:
            assert_kernel(g, kernel, i)


def test_scenario_sweep_with_extreme_overrides(ctx):
    base = cluster(256, 2048, [1, 2], seed=5)
    P, N = base.n_parts, base.n_nodes
    rng = np.random.default_rng(5)
    one = np.ones(8, np.uint8)
    heavy = rng.choice(P, 8, replace=False).astype(np.int32)
    w = np.where(base.part_has_weight > 0, np.abs(base.part_weight), 1).astype(np.int64)
    big = int(min(999999999, (I32_MAX // base.n_slots - (w.sum() - w[heavy[:2]].sum())) // 2))
    scs, opts = [], []
    variants = [
        {},
        dict(state_stickiness=np.array([I32_MAX, I32_MAX], np.int32), state_has_stickiness=np.ones(2, np.uint8)),
        dict(state_stickiness=np.array([-5, 0], np.int32), state_has_stickiness=np.ones(2, np.uint8)),
        dict(has_part_weights=1, weight_overrides=(heavy, np.array([-10**6, 0, 0, -1, -7, 0, -10**5, 0], np.int32), one)),
        dict(has_part_weights=1, weight_overrides=(heavy[:2], np.array([big, -big], np.int32), one[:2])),
        dict(has_part_weights=0),
    ]
    node_weights = [None, np.full(N, I32_MAX, np.int32), rng.choice([I32_MIN, -3, 0, 1], N).astype(np.int32)]
    for i, o in enumerate(variants):
        for j, nw in enumerate(node_weights):
            sc = dict(node_removed=base.node_removed.copy(), node_added=base.node_added.copy(), add_is_nil=0)
            if nw is not None:
                sc.update(has_node_weights=1, node_weight=nw, node_has_weight=np.ones(N, np.uint8))
            scs.append(sc)
            opts.append(o)
    base.booster_kind = blance_b200.BOOSTER_CBGT_MAX
    check_against_oracle(ctx, base, scs, opts, True)
