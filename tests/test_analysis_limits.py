"""The analysis judges at the limits the ABI accepts, and where the argument checks draw those limits: the map audit,
the exposure and the schedule oracles at 8 states, 32 slots in several layouts, 64 ops per partition and fault-domain
forests exactly 16 edges deep; blance_map_audit and blance_plan_scenarios_exposure refusing one past each limit and
accepting the limit itself, with no device.  The limit-size generators here also feed
tests/test_analysis_limits_gpu.py."""
import ctypes

import numpy as np
import pytest

import audit_oracle as AO
import audit_util as U
import exposure_oracle as EO
import schedule_oracle as SO
from test_exposure_oracle import calc_moves

from blance_b200 import abi as api
from blance_b200 import tables

INVALID, UNSUPPORTED, CUDA = -1, -2, -3
DEPTH = 16                                     # edges from a vertex to its root (AUDIT_DEPTH_MAX)

# 32-slot layouts: slot widths per state, with zero-width states before, between and after others
LAYOUTS = {"8x4": [4] * 8, "16+16": [16, 16], "1+31": [1, 31], "holes": [5, 0, 7, 0, 0, 12, 8, 0],
           "lead": [0, 8, 0, 8, 0, 8, 0, 8]}


def slot_off_of(widths):
    return np.concatenate([[0], np.cumsum(widths)]).astype(np.int32)


# ---- generators -------------------------------------------------------------------------------------------------

def deep_forest(NU, trees=1, depth=DEPTH, pad=0):
    """parent [NU + n_domains]: `trees` trees, each a spine of depth - 1 inner vertices from its root down, then two
    sibling vertices at depth - 1 under the spine's end; node i hangs under tree i % trees, sibling (i // trees) % 2,
    exactly `depth` edges below its root.  Copies under one sibling meet there, copies under both meet one level up,
    copies in two trees meet nowhere.  `pad` isolated inner vertices follow."""
    inner, leaf_parent = [], []
    for _ in range(trees):
        base = NU + len(inner)
        inner += [-1] + [base + d for d in range(depth - 2)]         # spine: depths 0 .. depth - 2
        end = base + depth - 2
        inner += [end, end]                                          # the two siblings at depth - 1
        leaf_parent.append((end + 1, end + 2))
    parent = [leaf_parent[i % trees][(i // trees) % 2] for i in range(NU)]
    return np.asarray(parent + inner + [-1] * pad, np.int32)


def forest_roots(NU, trees=1, depth=DEPTH):
    """The root of each tree of deep_forest(NU, trees, depth)."""
    return [NU + k * (depth + 1) for k in range(trees)]


def depths(parent):
    d = np.zeros(len(parent), np.int64)
    for v in range(len(parent)):
        u = int(parent[v])
        while u >= 0:
            d[v] += 1
            u = int(parent[u])
            assert d[v] <= 64
    return d


def forest_dict(parent, names):
    """The forest as {vertex: parent} names (the audit oracle's domain_parents) and the vertex names."""
    vnames = list(names) + ["dom%05d" % j for j in range(len(parent) - len(names))]
    return {vnames[v]: vnames[int(p)] for v, p in enumerate(parent) if p >= 0}, vnames


def limit_map(rng, widths, P, NU, full=0.5, dup=0.1, odd_shapes=0.08):
    """rows [P][32] and shape [P][S] over NU node ids: each list full to its last slot with probability `full`, else
    cut anywhere (a gap); a few nil and absent states; with probability `dup` a node listed twice in one row."""
    off = slot_off_of(widths)
    S, SL = len(widths), int(off[-1])
    rows = np.full((P, SL), -1, np.int32)
    shape = np.full((P, S), 2, np.uint8)
    for p in range(P):
        pool = rng.permutation(NU)[:SL] if NU >= SL else rng.integers(0, NU, SL)
        for s in range(S):
            u = rng.random()
            if u < odd_shapes:
                shape[p, s] = 0 if u < odd_shapes / 2 else 1
                continue
            w = widths[s]
            n = w if rng.random() < full else int(rng.integers(0, w + 1))
            rows[p, off[s]:off[s] + n] = pool[off[s]:off[s] + n]
        if rng.random() < dup:
            i, j = rng.choice(SL, 2, replace=False)
            if rows[p, i] >= 0 and rows[p, j] >= 0:
                rows[p, j] = rows[p, i]
    return rows, shape


def audit_tables(widths, cons, N, P, extra_ids=0):
    """PlanTables of an audit: states s0 .. s(S-1) in priority order (top = s0), `widths` slots per state."""
    S = len(widths)
    t = tables.PlanTables(N, S, P, list(range(S)), list(cons), n_node_ids=N + extra_ids)
    t.state_slot_off = slot_off_of(widths)
    t.n_slots = int(t.state_slot_off[-1])
    return t


def limit_constraints(rng, widths, kmax=16):
    """A constraint per state: up to min(width, kmax), at least one state constrained."""
    k = [int(rng.integers(0, min(w, kmax) + 1)) if rng.random() < 0.5 else min(w, kmax) for w in widths]
    if not any(k):
        k[int(np.argmax(widths))] = min(max(widths), kmax)
    return k


def expo_case(rng, widths, P, NN, full=0.6, dup=0.15, same=0.1):
    """(slot_off, beg, end, constraints, top) of a rebalance at a 32-slot layout: rows from limit_map (no nil or
    absent states in a move list), constraints up to 16, top in {-1, 0, S - 1}."""
    S = len(widths)
    beg, _ = limit_map(rng, widths, P, NN, full, dup, 0)
    end, _ = limit_map(rng, widths, P, NN, full, 0, 0)
    keep = rng.random(P) < same                                        # partitions without ops
    end[keep] = beg[keep]
    cons = rng.integers(0, 17, S).astype(np.int32)
    top = int(rng.choice([-1, 0, S - 1]))
    return slot_off_of(widths), beg, end, cons, top


def rows_64_ops(rng, widths, P, NN):
    """beg and end rows full to slot 31 whose 64 entries are 64 distinct nodes: CalcPartitionMoves gives each
    partition 32 adds and 32 dels, the most it emits."""
    assert NN >= 64
    beg = np.zeros((P, 32), np.int32)
    end = np.zeros((P, 32), np.int32)
    for p in range(P):
        perm = rng.permutation(NN)[:64]
        beg[p], end[p] = perm[:32], perm[32:]
    return slot_off_of(widths), beg, end


def cross_tree_rows(rng, widths, P, NU, trees=2):
    """beg rows on tree 0's nodes and end rows on tree 1's (deep_forest(NU, 2)), so every partition's deepest common
    ancestor walks from one tree, through none, into the other: chains of 17 vertices on both sides."""
    off = slot_off_of(widths)
    a, b = np.arange(0, NU, trees), np.arange(1, NU, trees)
    beg = np.full((P, int(off[-1])), -1, np.int32)
    end = beg.copy()
    for p in range(P):
        for rows, pool in ((beg, a), (end, b)):
            pick = rng.permutation(pool)
            for s, w in enumerate(widths):
                n = int(rng.integers(1 if w else 0, w + 1))
                rows[p, off[s]:off[s] + n] = pick[off[s]:off[s] + n]
    return off, beg, end


def expo_both(slot_off, beg, end, favor, cons, top, NN, count, parent=None, oracles=(EO.replay, EO.vectorised)):
    """The moves of beg -> end scheduled at `count`, through each exposure oracle."""
    moves = calc_moves(slot_off, beg, end, favor)
    ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], NN, count)
    return moves, [o(slot_off, beg, *moves, ro, so, cons, top, NN, parent) for o in oracles]


# ---- the generators reach the limits ----------------------------------------------------------------------------

def test_generators_reach_the_limits():
    for widths in LAYOUTS.values():
        assert sum(widths) == 32
    for trees in (1, 2):
        par = deep_forest(40, trees)
        d = depths(par)
        roots = forest_roots(40, trees)
        assert (d[:40] == DEPTH).all() and d.max() == DEPTH and (par[roots] == -1).all() and (par == -1).sum() == trees
    assert depths(deep_forest(8, 1, DEPTH + 1))[:8].max() == DEPTH + 1
    rng = np.random.default_rng(1)
    slot_off, beg, end = rows_64_ops(rng, LAYOUTS["8x4"], 20, 80)
    off, node, state, kind = calc_moves(slot_off, beg, end, True)
    assert (np.diff(off) == 64).all()
    rows, shape = limit_map(rng, LAYOUTS["holes"], 400, 50)
    assert (rows[:, 31] >= 0).any() and (rows[:, 31] == -1).any() and (shape == 0).any() and (shape == 1).any()


# ---- the exposure oracles ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_exposure_oracles_agree_at_32_slots(layout):
    rng = np.random.default_rng(sorted(LAYOUTS).index(layout) + 90)
    widths = LAYOUTS[layout]
    for trial in range(4):
        NN = int(rng.integers(34, 70))
        slot_off, beg, end, cons, top = expo_case(rng, widths, 24, NN)
        parent = deep_forest(NN, 1 + trial % 2) if trial % 3 else None
        for favor in (False, True):
            for c in (1, 2, 4):
                _, (lit, vec) = expo_both(slot_off, beg, end, favor, cons, top, NN, c, parent)
                EO.assert_equal(vec, lit, (layout, trial, favor, c))
    # bit 31 of a beg row is live somewhere: the last slot of a full row holds an entry
    assert (beg[:, 31] >= 0).any()


@pytest.mark.parametrize("trees", [1, 2])
def test_exposure_oracles_agree_on_64_ops_and_16_edge_forests(trees):
    rng = np.random.default_rng(trees)
    NN = 80
    parent = deep_forest(NN, trees)
    for widths in (LAYOUTS["8x4"], LAYOUTS["16+16"]):
        slot_off, beg, end = rows_64_ops(rng, widths, 10, NN)
        S = len(widths)
        cons = np.full(S, 16 if S == 2 else 4, np.int32)
        for favor in (False, True):
            for c in (1, 64):
                _, (lit, vec) = expo_both(slot_off, beg, end, favor, cons, 0, NN, c, parent)
                EO.assert_equal(vec, lit, (trees, S, favor, c))


def test_exposure_oracles_agree_when_copies_cross_trees():
    """Every copy moves from one 16-edge tree into the other; the roots' peaks are the partitions alone in a tree."""
    rng = np.random.default_rng(5)
    NU = 64
    parent = deep_forest(NU, 2)
    roots = forest_roots(NU, 2)
    widths = LAYOUTS["8x4"]
    slot_off, beg, end = cross_tree_rows(rng, widths, 12, NU)
    cons = np.full(8, 2, np.int32)
    for favor in (False, True):
        for c in (1, 3):
            _, (lit, vec) = expo_both(slot_off, beg, end, favor, cons, 7, NU, c, parent)
            EO.assert_equal(vec, lit, (favor, c))
            assert lit["dom_peak"][roots[0]] == 12 and lit["dom_peak_round"][roots[0]] == 0
            assert lit["dom_peak"][roots[1]] == 12 and lit["dom_peak_round"][roots[1]] > 0


def test_vectorised_dca_at_exactly_16_edges():
    """_dca clips chains at 17 vertices: a depth-16 node's chain reaches its root, and two copies under the two
    deepest siblings meet one level above them."""
    NU = 4
    parent = deep_forest(NU, 1)
    paths = EO._paths(NU, parent)
    assert paths[0, DEPTH] == NU and paths[0, DEPTH - 1] != -1          # leaf first: the root is entry 16
    nodes = np.array([[0, 2, -1], [0, 1, -1], [3, -1, -1]], np.int64)    # 0 and 2: one sibling; 0 and 1: both
    got = EO._dca(nodes, NU, paths)
    assert got.tolist() == [int(parent[0]), int(parent[parent[0]]), 3]


# ---- the schedule oracle ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("count", [1, 2, 64])
def test_schedule_oracle_equals_the_go_reading_on_64_op_partitions(count):
    rng = np.random.default_rng(count)
    NN = 96
    slot_off, beg, end = rows_64_ops(rng, LAYOUTS["16+16"], 12, NN)
    for favor in (False, True):
        off, node, state, kind = calc_moves(slot_off, beg, end, favor)
        assert int(np.diff(off).max()) == 64
        mover = None if favor else (rng.random(NN) >= 0.1).astype(np.uint8)
        ro, so, sc = SO.schedule(off, node, kind, NN, count, mover)
        want_ro, want_so = SO.flatten(SO.go_reading(off, node, kind, NN, count, mover))
        assert np.array_equal(ro, want_ro) and np.array_equal(so, want_so), (count, favor)


# ---- the audit oracle -------------------------------------------------------------------------------------------

def numpy_nodes_audit(t, rows, shape):
    """The nodes-only fields of the audit counted directly: short / over slots, dom_top / dom_all / dom_copies over
    node ids, the failover matrix."""
    P, S, N, NU = t.n_parts, t.n_states, t.n_nodes, t.n_node_ids
    off = np.asarray(t.state_slot_off)
    cons = np.asarray(t.state_constraints)
    listed = np.zeros(rows.shape, bool)                  # entries of list states before their first -1
    short, over = np.zeros(S, np.int64), np.zeros(S, np.int64)
    for s in range(S):
        lo, hi = int(off[s]), int(off[s + 1])
        if hi > lo:
            listed[:, lo:hi] = np.cumprod(rows[:, lo:hi] != -1, axis=1).astype(bool) & (shape[:, s] == 2)[:, None]
        n = listed[:, lo:hi].sum(axis=1)
        present = shape[:, s] != 0
        if cons[s] > 0:
            short[s] = np.maximum(cons[s] - n, 0)[present].sum()
            over[s] = np.maximum(n - cons[s], 0)[present].sum()
    copies = np.bincount(rows[listed], minlength=NU)
    lo, hi = int(off[0]), int(off[1])
    has_top = (shape[:, 0] == 2) & (hi > lo) & listed[:, lo] if hi > lo else np.zeros(P, bool)
    h = np.where(has_top, rows[:, lo] if hi > lo else -1, -1)
    dom_top = np.bincount(h[h >= 0], minlength=NU)
    first = np.where(listed.any(axis=1), rows[np.arange(P), np.argmax(listed, axis=1)], -1)
    alone = listed.any(axis=1) & np.where(listed, rows == first[:, None], True).all(axis=1)
    dom_all = np.bincount(first[alone], minlength=NU)
    n2n = np.zeros((N, N), np.int32)
    sel = listed & (h[:, None] >= 0) & (h[:, None] < N) & (rows < N) & (rows != h[:, None])
    pp, cc = np.nonzero(sel)
    np.add.at(n2n, (h[pp], rows[pp, cc]), 1)
    return dict(short_slots=short, over_slots=over, dom_top=dom_top, dom_all=dom_all, dom_copies=copies, n2n=n2n)


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_audit_oracle_equals_numpy_at_8_states_and_32_slots(layout):
    rng = np.random.default_rng(sorted(LAYOUTS).index(layout) + 300)
    widths = LAYOUTS[layout]                             # "lead": the top state has no slot, no partition a primary
    for trial in range(3):
        N = int(rng.integers(20, 60))
        extra = int(rng.integers(0, 3))
        t = audit_tables(widths, limit_constraints(rng, widths), N, 300, extra)
        rows, shape = limit_map(rng, widths, t.n_parts, N + extra)
        names = U.node_names(t)
        e = U.expected(t, U.oracle_of(t, rows, shape, names), names)
        want = numpy_nodes_audit(t, rows, shape)
        for f in ("short_slots", "over_slots", "dom_top", "dom_all", "dom_copies", "n2n"):
            assert np.array_equal(e[f], want[f]), (layout, trial, f)
        assert e["short_parts"] > 0 and e["dom_copies"].sum() > 0


def test_audit_oracle_walks_16_edges_and_refuses_17():
    NU = 6
    names = ["n%04d" % i for i in range(NU)]
    dp, vnames = forest_dict(deep_forest(NU, 2), names)
    root0 = vnames[NU]
    pmap = {"p0": {"s0": ["n0000"], "s1": ["n0002"]}, "p1": {"s0": ["n0000"], "s1": ["n0001"]}}
    r = AO.audit(pmap, {"s0": (0, 1), "s1": (1, 1)}, names, domain_parents=dp)
    assert r["dom_all"][root0] == 1 and r["dom_copies"][root0] == 3      # p1 spans both trees
    deep, _ = forest_dict(deep_forest(NU, 1, DEPTH + 1), names)
    with pytest.raises(AssertionError, match="deeper than 16"):
        AO.audit(pmap, {"s0": (0, 1), "s1": (1, 1)}, names, domain_parents=deep)


# ---- one past each limit, without a device ----------------------------------------------------------------------

def past_the_checks(st, msg):
    """What a call whose arguments all pass returns without a context: BLANCE_ERR_CUDA on a machine without a
    device, "ctx is NULL" on one with a device."""
    return (st == CUDA and "no CUDA device" in msg) or (st == INVALID and "ctx is NULL" in msg)


def audit_call(t, parent=None):
    lib = api.capi()
    s = t.struct()
    o = api.AuditOpts()
    keep = None
    if parent is not None:
        keep = np.ascontiguousarray(parent, np.int32)
        o.domain_parent, o.n_domains = keep.ctypes.data, keep.size - t.n_node_ids
    r = tables.AuditResult(t, int(t.n_rules) if t.has_hier_rules else 0)
    rows = np.ascontiguousarray(t.cur_rows, np.int32)
    shape = np.ascontiguousarray(t.cur_shape, np.uint8)
    st = lib.blance_map_audit(None, ctypes.byref(s), rows.ctypes.data if rows.size else None,
                              shape.ctypes.data if shape.size else None, ctypes.byref(o), ctypes.byref(r.out))
    return st, lib.blance_last_error(None).decode()


def small_audit(S=2, widths=None, N=6):
    widths = widths or [1] * S
    t = audit_tables(widths, [1] * S, N, 4)
    t.cur_rows = np.full((4, t.n_slots), -1, np.int32)
    t.cur_rows[:, 0] = np.arange(4)
    t.cur_shape = np.full((4, S), 2, np.uint8)
    return t


def with_rules(t, n_rules, n_bits):
    t.has_hier_rules, t.n_rules, t.n_hier_bits = 1, n_rules, n_bits
    per, rem = divmod(n_rules, t.n_states)
    t.rule_off = np.concatenate([[0], np.cumsum([per + (s < rem) for s in range(t.n_states)])]).astype(np.int32)
    t.ie_mask = np.zeros(n_rules * (t.n_node_ids + 1) * ((n_bits + 31) // 32), np.uint32)
    return t


def test_map_audit_forest_depth_limit():
    t = small_audit()
    assert past_the_checks(*audit_call(t, deep_forest(6, 1))), audit_call(t, deep_forest(6, 1))
    assert past_the_checks(*audit_call(t, deep_forest(6, 2)))
    st, msg = audit_call(t, deep_forest(6, 1, DEPTH + 1))
    assert st == INVALID and "16 edges" in msg, msg


def test_map_audit_state_and_slot_limits():
    assert past_the_checks(*audit_call(small_audit(8, [4] * 8, N=40)))
    st, msg = audit_call(small_audit(9, [4] * 8 + [0], N=40))
    assert st == UNSUPPORTED and "8 model states" in msg, msg
    st, msg = audit_call(small_audit(8, [4] * 7 + [5], N=40))
    assert st == UNSUPPORTED and "32 slots" in msg, msg


def test_map_audit_rule_and_bit_limits():
    # 256 rules over 4 096 bits pass the checks; one more rule or one more bit does not
    assert past_the_checks(*audit_call(with_rules(small_audit(8, [4] * 8, N=40), 256, 4096)))
    st, msg = audit_call(with_rules(small_audit(8, [4] * 8, N=40), 257, 4096))
    assert st == UNSUPPORTED and "256" in msg, msg
    st, msg = audit_call(with_rules(small_audit(8, [4] * 8, N=40), 256, 4097))
    assert st == UNSUPPORTED and "4096" in msg, msg


def scenario_exposure_call(t, parent):
    """blance_plan_scenarios_exposure with a NULL context, one scenario of the base, one count, dom peaks, the
    forest `parent`."""
    lib = api.capi()
    base = t.struct()
    sc = (api.Scenario * 1)()
    sc[0].node_removed, sc[0].node_added = base.node_removed, base.node_added
    out, sched = (api.ScenarioOut * 1)(), (api.ScenarioScheduleOut * 1)()
    counts = (ctypes.c_int32 * 1)(1)
    par = np.ascontiguousarray(parent, np.int32)
    peaks = np.zeros(par.size, np.int64)
    ex = (api.ExposureOut * 1)()
    ex[0].dom_peak = peaks.ctypes.data
    eopts = api.AuditOpts(0, par.size - t.n_node_ids, par.ctypes.data)
    st = lib.blance_plan_scenarios_exposure(None, ctypes.byref(base), 1, sc, None, 0, 0, 1, counts, None, out, sched, None,
                                            None, ctypes.byref(eopts), 4, ex)
    return st, lib.blance_last_error(None).decode()


def scenario_base(widths, N=40):
    S = len(widths)
    t = tables.PlanTables(N, S, 6, list(range(S)), [min(w, 1) for w in widths])
    t.state_slot_off = slot_off_of(widths)
    t.n_slots = int(t.state_slot_off[-1])
    t.prev_rows = np.full((6, t.n_slots), -1, np.int32)
    t.prev_rows[:, 0] = np.arange(6)
    t.cur_rows = t.prev_rows.copy()
    t.prev_shape = np.full((6, S), 2, np.uint8)
    t.cur_shape = t.prev_shape.copy()
    t.part_in_prev[:] = 1
    return t


def test_scenario_exposure_forest_depth_limit():
    t = scenario_base(LAYOUTS["8x4"])
    for trees in (1, 2):
        assert past_the_checks(*scenario_exposure_call(t, deep_forest(t.n_node_ids, trees)))
    st, msg = scenario_exposure_call(t, deep_forest(t.n_node_ids, 1, DEPTH + 1))
    assert st == INVALID and "16 edges" in msg, msg
