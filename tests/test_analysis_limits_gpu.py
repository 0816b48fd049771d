"""The analysis kernels at the limits the ABI accepts, each against its oracle field for field: the map audit at 8 states
and 32 slots, 256 rules, hierarchy universes up to 4 096 bits, 16-edge forests, both sides of the shared-memory switch
and an 8 192-node failover matrix; the exposure of a handle at 32-slot rows, 64 ops per partition, copies crossing
between two 16-edge trees, series on both sides of the 512-entry scan chunks and 8 192 node ids; scenario waves on both
sides of the summary's shared-memory switch, at 8 states x 4 constraints with rules and a deep forest, and wider than
65 535 scenarios in one call.  Needs an H100; run with -m gpu."""
import re

import numpy as np
import pytest

import audit_util as U
import exposure_oracle as EO
import scenario_exposure_ref as REF
import schedule_oracle as SO
from test_analysis_limits import (DEPTH, LAYOUTS, audit_tables, cross_tree_rows, deep_forest, expo_case, forest_dict,
                                  forest_roots, limit_constraints, limit_map, numpy_nodes_audit, rows_64_ops)
from test_exposure_gpu import device_and
from test_scenario_audit_gpu import final_map, flat
from test_scenario_schedule import assert_same_summaries, schedule_summaries
from test_scenario_schedule_gpu import default_mover, got_summaries, move_lists
from test_scenarios_gpu import _node_failures, assert_scenario, check_against_oracle, oracle_tables, reference_summary

from blance_b200 import synth, tables
from blance_b200.abi import BlanceError

pytestmark = pytest.mark.gpu
BIG = 1 << 12                                   # a series cap above any R of the scenario waves here


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


# ---- the map audit ----------------------------------------------------------------------------------------------

def rack_hierarchy(names, rack=4, zone=4):
    """node -> rack -> zone -> root over `names` (the rules' NodeHierarchy)."""
    parents = {n: "rack%03d" % (i // rack) for i, n in enumerate(names)}
    for r in sorted(set(parents.values())):
        parents[r] = "zone%03d" % (int(r[4:]) // zone)
    for z in sorted(v for v in set(parents.values()) if v.startswith("zone")):
        parents[z] = "root"
    return parents


def audit_check(ctx, t, rows, shape, names, parents=None, rules=None, parent=None, rule_modes=(False, True),
                forest_modes=(False, True)):
    """blance_map_audit against the string-map oracle with and without the rules, the forest and the failover
    matrix, as test_audit_gpu.check.  Returns the oracle's arrays of the last combination."""
    dparents, vnames = forest_dict(parent, names) if parent is not None else (None, names)
    for with_rules in rule_modes:
        if with_rules:
            U.set_hierarchy(t, parents, rules, names)
        else:
            t.has_hier_rules, t.n_rules = 0, 0
        for with_forest in forest_modes:
            e = U.expected(t, U.oracle_of(t, rows, shape, names, parents, rules, dparents if with_forest else None), names,
                           vnames if with_forest else names)
            for n2n in (False, True):
                got = ctx.map_audit(t, rows, shape, n2n=n2n, domain_parent=parent if with_forest else None)
                U.assert_audit(got, e, n2n, (with_rules, with_forest, n2n))
    return e


@pytest.mark.parametrize("layout", ["8x4", "16+16"])
def test_audit_at_32_slots_with_rules_on_every_state(ctx, layout):
    rng = np.random.default_rng(11)
    widths = LAYOUTS[layout]
    cons = [4] * 8 if layout == "8x4" else [16, 16]
    N = 48
    t = audit_tables(widths, cons, N, 500, 2)
    rows, shape = limit_map(rng, widths, t.n_parts, N + 2, full=0.6)
    names = U.node_names(t)
    parents = rack_hierarchy(names)
    rules = {"s%d" % s: [(1, 0), (2, 1), (3, 1)] for s in range(len(widths))}
    e = audit_check(ctx, t, rows, shape, names, parents, rules, deep_forest(N + 2, 2))
    assert e["rule_miss_parts"] > 0 and e["short_parts"] > 0
    if layout == "16+16":
        # every position 0 .. 15 of state s1 is tested: each full s1 list adds 16 tests to each of its rules
        n = np.minimum(np.cumprod(rows[:, 16:] != -1, axis=1).sum(axis=1), 16)[shape[:, 1] == 2]
        assert (n == 16).any()
        assert (e["rule_tested"][t.rule_off[1]:t.rule_off[2]] == n.sum()).all()


def test_audit_with_256_rules(ctx):
    rng = np.random.default_rng(12)
    widths = [4] * 8
    N = 40
    t = audit_tables(widths, [1] * 8, N, 300)
    rows, shape = limit_map(rng, widths, t.n_parts, N, full=0.7)
    names = U.node_names(t)
    pairs = [(i, x) for i in range(4) for x in range(3)]
    rules = {"s%d" % s: [pairs[(s + j) % len(pairs)] for j in range(32)] for s in range(8)}
    e = audit_check(ctx, t, rows, shape, names, rack_hierarchy(names), rules, forest_modes=(False,))
    assert t.n_rules == 256 and e["rule_tested"][-32:].sum() > 0 and e["rule_miss"][-32:].sum() > 0


def wide_universe(rng, N, extra, P, rack=32, zone=4):
    """A hierarchy over N nodes plus `extra` leaves outside nodesAll (racks of `rack` leaves, the extras in the last
    zone), rules whose include and exclude sets reach the last mask words, and a 2-state map whose primaries sit on
    the highest nodes half the time, with replicas in the primary's rack, zone or anywhere."""
    t = audit_tables([1, 3], [1, 3], N, P)
    names = U.node_names(t)
    leaves = names + ["g%03d" % i for i in range(extra)]
    parents = rack_hierarchy(leaves, rack, zone)
    rules = {"s1": [(1, 0), (2, 1)], "s0": [(1, 0)]}
    rows = np.full((P, 4), -1, np.int32)
    shape = np.full((P, 2), 2, np.uint8)
    hi = max(0, N - 1024)
    for p in range(P):
        h = int(rng.integers(hi, N)) if rng.random() < 0.5 else int(rng.integers(0, N))
        rows[p, 0] = h
        r0 = h - h % rack
        for j in range(1, 4):
            u = rng.random()
            if u < 0.4:
                x = int(rng.integers(r0, min(N, r0 + rack)))
            elif u < 0.7:
                z0 = h - h % (rack * zone)
                x = int(rng.integers(z0, min(N, z0 + rack * zone)))
            else:
                x = int(rng.integers(0, N))
            rows[p, j] = x
        if rng.random() < 0.1:
            shape[p, 0] = int(rng.integers(0, 2))         # no primary: positions after the first restart there
        if rng.random() < 0.1:
            rows[p, 1 + int(rng.integers(0, 3))] = -1
    return t, rows, shape, names, parents, rules


@pytest.mark.parametrize("N,extra", [(33, 0), (65, 0), (97, 0), (4000, 96)])
def test_audit_hierarchy_universes(ctx, N, extra):
    rng = np.random.default_rng(N)
    t, rows, shape, names, parents, rules = wide_universe(rng, N, extra, 600 if N < 4000 else 1500, rack=8 if N < 4000 else 32)
    e = audit_check(ctx, t, rows, shape, names, parents, rules, rule_modes=(True,), forest_modes=(False,))
    assert t.n_hier_bits == N + extra and t.hier_words == (N + extra + 31) // 32
    assert e["rule_miss_parts"] > 0 and e["rule_tested"].sum() > e["rule_miss"].sum()
    if N == 4000:
        mask = t.ie_mask.reshape(t.n_rules, t.n_node_ids + 1, t.hier_words)
        assert mask[:, :, 96:].any() and mask[:, :, 125:].any()           # words of rv[3], the extras' last words
        tested_high = (rows[:, 1:] >= 3072) & (shape[:, 1:2] == 2)
        assert tested_high.sum() > 100


def test_audit_forest_16_edges_two_trees(ctx):
    rng = np.random.default_rng(16)
    widths = LAYOUTS["8x4"]
    N = 64
    t = audit_tables(widths, limit_constraints(rng, widths), N, 600)
    rows, shape = limit_map(rng, widths, t.n_parts, N, full=0.5)
    # a third of the partitions in tree 0 only, a third under one deepest vertex only
    pools = [np.arange(0, N, 2), np.arange(0, N, 4)]
    for p in range(t.n_parts // 3 * 2):
        pool = pools[p % 2]
        sel = rows[p] >= 0
        rows[p, sel] = rng.choice(pool, int(sel.sum()))
    parent = deep_forest(N, 2)
    names = U.node_names(t)
    e = audit_check(ctx, t, rows, shape, names, parent=parent, rule_modes=(False,))
    roots = forest_roots(N, 2)
    assert e["dom_all"][roots[0]] > 0 and e["dom_top"][roots[0]] > 0 and e["dom_copies"][roots].sum() == e["dom_copies"][:N].sum()
    # node 0's parent is one of tree 0's two deepest inner vertices; copies under both meet one level up
    assert e["dom_all"][parent[0]] > 0 and e["dom_all"][parent[parent[0]]] > e["dom_all"][parent[0]]


@pytest.mark.parametrize("V", [3754, 3755])
def test_audit_domain_tables_at_the_shared_memory_switch(ctx, V):
    """3 x 4 x V bytes <= 44 KiB: V = 3 754 keeps the per-vertex tables in shared memory, 3 755 does not."""
    rng = np.random.default_rng(3754)
    widths = LAYOUTS["holes"]
    N = 60
    t = audit_tables(widths, limit_constraints(rng, widths), N, 800)
    rows, shape = limit_map(rng, widths, t.n_parts, N)
    base = deep_forest(N, 2)
    parent = deep_forest(N, 2, pad=V - len(base))
    assert len(parent) == V
    audit_check(ctx, t, rows, shape, U.node_names(t), parent=parent, rule_modes=(False,), forest_modes=(True,))


def test_audit_failover_matrix_at_8192_nodes(ctx):
    """The largest matrix entry, tied between (3, 5) and (8 191, 8 190): the lowest index wins."""
    rng = np.random.default_rng(8192)
    N, P, tie = 8192, 40000, 9
    t = audit_tables([1, 2], [1, 2], N, P)
    rows = rng.integers(0, N, (P, 3)).astype(np.int32)
    rows[:tie] = [3, 5, -1]
    rows[tie:2 * tie] = [8191, 8190, -1]
    shape = np.full((P, 2), 2, np.uint8)
    got = ctx.map_audit(t, rows, shape, n2n=True)
    want = numpy_nodes_audit(t, rows, shape)
    for f in ("short_slots", "over_slots", "dom_top", "dom_all", "dom_copies"):
        assert np.array_equal(getattr(got, f), want[f]), f
    assert np.array_equal(got.n2n, want["n2n"])
    assert want["n2n"].max() == tie and want["n2n"][3, 5] == want["n2n"][8191, 8190] == tie
    assert got.n2n_max == (tie, 3, 5)


# ---- the exposure of a handle -----------------------------------------------------------------------------------

@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_exposure_random_32_slot_lists(ctx, layout):
    rng = np.random.default_rng(sorted(LAYOUTS).index(layout) + 50)
    widths = LAYOUTS[layout]
    for trial in range(4):
        NN = int(rng.integers(34, 80))
        slot_off, beg, end, cons, top = expo_case(rng, widths, 40, NN)
        parent = deep_forest(NN, 1 + trial % 2) if trial % 2 else None
        h, total = ctx.moves_create(slot_off, beg, end, trial % 2 == 0, NN)
        for c in (1, 2, 4):
            device_and(ctx, EO.replay, slot_off, beg, h, total, c, cons, top, NN, parent)
        ctx.moves_free(h)
    assert (beg[:, 31] >= 0).any()


def test_exposure_64_ops_per_partition(ctx):
    rng = np.random.default_rng(64)
    NN = 200
    for widths, P, oracle in ((LAYOUTS["8x4"], 20, EO.replay), (LAYOUTS["16+16"], 1000, EO.vectorised)):
        slot_off, beg, end = rows_64_ops(rng, widths, P, NN)
        S = len(widths)
        cons = np.full(S, 16 if S == 2 else 4, np.int32)
        parent = deep_forest(NN, 2)
        for favor in (False, True):
            h, total = ctx.moves_create(slot_off, beg, end, favor, NN)
            assert total == 64 * P
            for c in (1, 64):
                device_and(ctx, oracle, slot_off, beg, h, total, c, cons, 0, NN, parent)
            ctx.moves_free(h)


def test_exposure_copies_cross_between_16_edge_trees(ctx):
    rng = np.random.default_rng(34)
    NU = 64
    parent = deep_forest(NU, 2)
    roots = forest_roots(NU, 2)
    for widths, P, oracle in ((LAYOUTS["8x4"], 24, EO.replay), (LAYOUTS["1+31"], 2000, EO.vectorised)):
        slot_off, beg, end = cross_tree_rows(rng, widths, P, NU)
        cons = np.full(len(widths), 1, np.int32)
        for favor in (False, True):
            h, total = ctx.moves_create(slot_off, beg, end, favor, NU)
            for c in (1, 3):
                got, _ = device_and(ctx, oracle, slot_off, beg, h, total, c, cons, len(widths) - 1, NU, parent)
                assert got["dom_peak"][roots].tolist() == [P, P]
                # every copy starts in tree A; tree B holds every partition once its last tree-A copy is gone
                assert got["dom_peak_round"][roots[0]] == 0 and 0 < got["dom_peak_round"][roots[1]] <= got["rounds"]
            ctx.moves_free(h)


def node0_series_case(R, last):
    """R rounds of one op each on node 0 at count 1: a adds (weight 3, scheduled first), b dels, and one promote
    (weight 1, the very first) when R - a - b = 1.  NO_COPY starts at a, falls to 0, climbs to b: last=False makes
    b = a, so the peak is first reached at round 0 and again at the last round; last=True makes b = a + 1, so the
    peak is first reached at the last entry."""
    a = (R - 1) // 2 if last else R // 2
    b = a + 1 if last else a
    promote = R - a - b
    P = a + b + promote + 5                                           # five partitions without ops
    beg = np.full((P, 2), -1, np.int32)
    end = beg.copy()
    end[:a, 0] = 0                                                    # add 0 as primary
    beg[a:a + b, 0] = 0                                               # del 0
    if promote:
        beg[a + b, 1] = 0
        end[a + b, 0] = 0
    beg[a + b + promote:, 0] = end[a + b + promote:, 0] = 0
    return np.array([0, 1, 2], np.int32), beg, end, a, b


@pytest.mark.parametrize("R1", [511, 512, 513, 1024, 1025])
@pytest.mark.parametrize("last", [False, True])
def test_exposure_series_across_scan_chunks(ctx, R1, last):
    slot_off, beg, end, a, b = node0_series_case(R1 - 1, last)
    h, total = ctx.moves_create(slot_off, beg, end, False, 1)
    got, sc = device_and(ctx, EO.vectorised, slot_off, beg, h, total, 1, np.array([1, 0], np.int32), 0, 1)
    ctx.moves_free(h)
    assert sc["rounds"] == R1 - 1 == got["rounds"]
    m = EO.METRICS.index("NO_COPY")
    series = np.concatenate([np.arange(a, -1, -1), np.arange(1, b + 1)])
    if R1 - 1 > a + b:
        series = np.concatenate([[a], series])                       # the promote's round changes no copy count
    assert np.array_equal(got["series"][m], series)
    assert got["peak"][m] == max(a, b) and got["area"][m] == series.sum()
    assert got["peak_round"][m] == (R1 - 1 if last else 0)
    c = EO.METRICS.index("COPIES")
    assert got["peak"][c] == a + b + 5 + (R1 - 1 > a + b) and got["peak_round"][c] == a + (R1 - 1 > a + b)


def test_exposure_8192_node_ids_with_a_forest(ctx):
    rng = np.random.default_rng(8193)
    NN = 8192
    parent = deep_forest(NN, 2)
    assert len(parent) > NN
    slot_off, beg, end, cons, top = expo_case(rng, LAYOUTS["8x4"], 2500, NN)
    h, total = ctx.moves_create(slot_off, beg, end, False, NN)
    for c in (1, 4):
        device_and(ctx, EO.vectorised, slot_off, beg, h, total, c, cons, top, NN, parent)
    ctx.moves_free(h)


def test_exposure_refuses_one_past_each_limit(ctx):
    rng = np.random.default_rng(9)
    NN = 40
    for widths, match in (([4] * 7 + [3, 1], "more than 8 states"), ([4] * 7 + [5], "more than 32 slots")):
        slot_off = np.concatenate([[0], np.cumsum(widths)]).astype(np.int32)
        beg, _ = limit_map(rng, widths, 10, NN, odd_shapes=0)
        end, _ = limit_map(rng, widths, 10, NN, odd_shapes=0)
        h, _ = ctx.moves_create(slot_off, beg, end, False, NN)
        ctx.moves_schedule(h, 1)
        with pytest.raises(BlanceError, match=match):
            ctx.moves_exposure(h, np.ones(len(widths), np.int32), 0)
        ctx.moves_free(h)
    slot_off, beg, end, cons, top = expo_case(rng, LAYOUTS["8x4"], 10, NN)
    h, total = ctx.moves_create(slot_off, beg, end, False, NN)
    ctx.moves_schedule(h, 1)
    with pytest.raises(BlanceError, match="16 edges"):
        ctx.moves_exposure(h, cons, top, deep_forest(NN, 1, DEPTH + 1))
    device_and(ctx, EO.replay, slot_off, beg, h, total, 1, cons, top, NN, deep_forest(NN, 1))
    ctx.moves_free(h)


# ---- scenario waves ---------------------------------------------------------------------------------------------

def summary_base(S, NU, P, seed):
    """A base of NU nodes, S states of constraint 1 and full rows: NU = node ids sizes the summary's tables."""
    rng = np.random.default_rng(seed)
    t = tables.PlanTables(NU, S, P, list(range(S)), [1] * S)
    rows = np.stack([rng.permutation(NU)[:S] for _ in range(P)]).astype(np.int32)
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:] = 2
    t.cur_shape[:] = 2
    t.part_in_prev[:] = 1
    t.max_iters = 3
    return t


@pytest.mark.parametrize("S,NU", [(1, 2048), (1, 2049), (2, 1536), (2, 1537), (8, 614), (8, 615)])
def test_scenario_summary_at_the_shared_memory_switch(ctx, S, NU):
    """16 NU + 8 S NU bytes <= 48 KiB keeps node_ops and state_node_load in shared memory; one node more does not."""
    t = summary_base(S, NU, 3000, NU)
    scs = _node_failures(t, [[], [0], list(range(1, 40))])
    check_against_oracle(ctx, t, scs, False)
    check_against_oracle(ctx, t, scs, True, max_concurrent=1)


def test_scenario_summary_8192_node_ids(ctx):
    wide = synth.make_rebalance(4, P=4096, N=8192)
    assert wide.n_node_ids >= 8192
    check_against_oracle(ctx, wide, _node_failures(wide, [[3]]), False)


def limit_scenario_base(seed):
    """8 states x 4 constraints (32 slots) over 72 nodes, rules on four states, every row full."""
    rng = np.random.default_rng(seed)
    N, P = 72, 400
    t = tables.PlanTables(N, 8, P, list(range(8)), [4] * 8)
    rows = np.stack([rng.permutation(N)[:32] for _ in range(P)]).astype(np.int32)
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:] = 2
    t.cur_shape[:] = 2
    t.part_in_prev[:] = 1
    t.max_iters = 4
    names = U.node_names(t)
    U.set_hierarchy(t, rack_hierarchy(names, 6, 3), {"s1": [(2, 1)], "s3": [(3, 2), (1, 0)], "s5": [(2, 0)], "s7": [(3, 1)]}, names)
    return t, rng


def test_scenario_wave_at_8_states_with_rules_and_a_deep_forest(ctx):
    t, rng = limit_scenario_base(8)
    parent = deep_forest(t.n_node_ids, 2)
    gone = np.zeros(t.n_node_ids, np.uint8)
    gone[t.prev_rows[0]] = 1                              # partition 0 loses all 32 of its nodes: 64 ops
    scs = [dict(node_removed=gone), dict(node_removed=(np.arange(t.n_node_ids) < 3).astype(np.uint8)), {}]
    counts = [1, 2, 64]
    mv = default_mover(t)
    for favor in (False, True):
        res = ctx.plan_scenarios(t, scs, favor, want_rows=range(len(scs)), schedule=counts,
                                 audit=dict(n2n=True, domain_parent=parent), exposure=dict(domain_parent=parent, series_cap=BIG))
        for i, (sc, r) in enumerate(zip(scs, res)):
            st = tables.scenario_tables(t, sc)
            ref = oracle_tables(st)
            assert_scenario(r, ref, reference_summary(st, ref.next_rows, ref.warn, favor), (favor, i))
            off, node, kind, _, _ = move_lists(st, r.next_rows, favor)
            if i == 0:
                assert int(np.diff(off)[0]) == 64
            rows, shape = final_map(st, r)
            assert flat(r.audit) == flat(ctx.map_audit(st, rows, shape, n2n=True, domain_parent=parent)), (favor, i)
            for k, c in enumerate(counts):
                ro, so, _ = SO.schedule(off, node, kind, st.n_node_ids, c, mv)
                assert_same_summaries(got_summaries(r.schedules[k]), schedule_summaries(off, node, st.n_node_ids, ro, so), (favor, i, c))
                want, _ = REF.scenario_exposure(st, r.next_rows, favor, c, domain_parent=parent)
                EO.assert_equal(r.exposures[k], want, (favor, i, c))
        assert res[0].audit.rule_tested.sum() > 0


def _tiny_base(P=12, N=8):
    rng = np.random.default_rng(3)
    t = tables.PlanTables(N, 2, P, [0, 1], [1, 1])
    rows = np.stack([rng.permutation(N - 2)[:2] for _ in range(P)]).astype(np.int32)
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:] = 2
    t.cur_shape[:] = 2
    t.part_in_prev[:] = 1
    t.max_iters = 3
    return t


def tiny_variants(t):
    """Every removal of at most two of nodes 0 .. 5, with nodes 6 / 7 added or not, add_is_nil, and two weight
    patterns: 352 distinct scenarios."""
    N = t.n_nodes
    out = []
    rms = [()] + [(a,) for a in range(6)] + [(a, b) for a in range(6) for b in range(a + 1, 6)]
    for rm in rms:
        for add in ((), (6,), (7,), (6, 7)):
            for nil in (0, 1):
                for hw in (0, 1):
                    r = np.zeros(N, np.uint8)
                    r[list(rm)] = 1
                    a = np.zeros(N, np.uint8)
                    a[list(add)] = 1
                    out.append(dict(node_removed=r, node_added=a, add_is_nil=nil, has_node_weights=hw,
                                    node_weight=np.array([1, 3, 1, 2, 1, 1, 4, 1], np.int32), node_has_weight=np.ones(N, np.uint8)))
    return out


def _waves(err):
    return [int(x) for x in re.findall(r"scenario wave at \d+: (\d+) scenarios", err)]


@pytest.mark.parametrize("with_schedule", [False, True])
def test_more_than_65535_scenarios_in_one_call(ctx, with_schedule, capfd, monkeypatch):
    t = _tiny_base()
    variants = tiny_variants(t)
    n = 70000
    pick = np.random.default_rng(7).integers(0, len(variants), n)
    scs = [variants[j] for j in pick]
    kw = dict(schedule=[1, 2], audit={}) if with_schedule else {}
    monkeypatch.setenv("BLANCE_SCENARIO_TIMES", "1")
    capfd.readouterr()
    res = ctx.plan_scenarios(t, scs, False, want_rows=range(n), **kw)
    waves = _waves(capfd.readouterr().err)
    assert sum(waves) == n and max(waves) <= 65535 and len(waves) >= 2, waves[:4]
    capped = ctx.plan_scenarios(t, scs, False, max_concurrent=4096, want_rows=range(n), **kw)
    assert sum(_waves(capfd.readouterr().err)) == n
    monkeypatch.delenv("BLANCE_SCENARIO_TIMES")
    _same(res, capped, with_schedule)
    # every scenario against the oracle of its variant, computed once per variant
    mv = default_mover(t)
    want = {}
    for j in np.unique(pick):
        st = tables.scenario_tables(t, variants[j])
        ref = oracle_tables(st)
        summ = reference_summary(st, ref.next_rows, ref.warn, False)
        sched = aud = None
        if with_schedule:
            off, node, kind, _, _ = move_lists(st, ref.next_rows, False)
            sched = [schedule_summaries(off, node, st.n_node_ids, *SO.schedule(off, node, kind, st.n_node_ids, c, mv)[:2]) for c in (1, 2)]
            names = U.node_names(st)
            r = type("R", (), dict(next_rows=ref.next_rows, next_shape=ref.next_shape))
            rows, shape = final_map(st, r)
            aud = U.expected(st, U.oracle_of(st, rows, shape, names), names)
        want[int(j)] = (ref, summ, sched, aud)
    for i, r in enumerate(res):
        ref, summ, sched, aud = want[int(pick[i])]
        assert_scenario(r, ref, summ, i)
        if with_schedule:
            for s, w in zip(r.schedules, sched):
                assert_same_summaries(got_summaries(s), w, i)
            U.assert_audit(r.audit, aud, False, i)


def _same(a, b, with_schedule):
    for i, (x, y) in enumerate(zip(a, b)):
        for f in ("next_rows", "next_shape", "warn", "node_ops", "state_node_load"):
            assert np.array_equal(getattr(x, f), getattr(y, f)), (i, f)
        assert (x.iters_run, x.converged, x.steps, x.parts_moved, x.ops_total, x.warn_parts) == \
            (y.iters_run, y.converged, y.steps, y.parts_moved, y.ops_total, y.warn_parts), i
        if with_schedule:
            for s, u in zip(x.schedules, y.schedules):
                assert_same_summaries(got_summaries(s), got_summaries(u), i)
            assert flat(x.audit) == flat(y.audit), i
