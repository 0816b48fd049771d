"""Parity tests proper: the CUDA path, called through the C ABI of
libblance_b200.so (directly, or underneath the C++ host mirror), against the
reference's golden vectors and against the CPU oracle on identical tables.
Integer/index work: the bar is bit-exact rows, shapes, warnings, iteration and step
counts.  Needs an H100; run with `-m gpu`."""
import copy
import ctypes

import numpy as np
import pytest

import golden_util as G
from oracle_loader import fast_lib_path, literal
from randgen import random_instance

import blance_b200
from blance_b200 import _host, synth, tables

pytestmark = pytest.mark.gpu

FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
FAST.oracle_fast_calc_partition_moves.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 4


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def oracle_tables(t):
    r = tables.PlanResult(t)
    s = t.struct()
    assert FAST.oracle_fast_plan_next_map(ctypes.byref(s), ctypes.byref(r.out)) == 0
    return r


def assert_same(got, ref):
    assert np.array_equal(got.next_rows, ref.next_rows)
    assert np.array_equal(got.next_shape, ref.next_shape)
    assert np.array_equal(got.warn, ref.warn)
    assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps)


# ---- the reference's own golden vectors through the product's string API -----------------

@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_plan_next_map_golden_gpu(c):
    kw = G.plan_kwargs(c)
    r = _host.PlanNextMapEx(**kw)
    assert r["next_map"] == G.pmap(c["exp"])
    assert G.count_warnings(c, r["warnings"]) == c["expNumWarnings"]


def test_caller_maps_are_mutated_like_plan_go_49_52():
    L = literal()
    for c in G.plan_cases():
        kw = G.plan_kwargs(c)
        lit = L.plan_next_map_ex(**copy.deepcopy(kw))
        r = _host.PlanNextMapEx(**kw)
        assert r["prev_map"] == lit["prev_map"], G.case_id(c)
        assert r["partitions_to_assign"] == lit["partitions_to_assign"], G.case_id(c)
        assert r["iterations"] == lit["iterations"], G.case_id(c)


def test_calc_partition_moves_golden_gpu():
    for c in G.load("moves_cases.json")["calcPartitionMoves"]:
        got = blance_b200.CalcPartitionMoves(c["states"], c["before"], c["after"], c["favorMinNodes"])
        assert len(got) == len(c["exp"]), c["index"]
        for op, e in zip(got, c["exp"]):
            assert op.Node == e["node"] and op.State == e["state"] and op.Op in e["op"], (c["index"], got, c["exp"])


def test_orchestrate_derived_move_sequences_gpu():
    for c in G.load("moves_cases.json")["orchestrateDerived"]:
        got = blance_b200.CalcPartitionMoves(c["states"], c["before"], c["after"], c["favorMinNodes"])
        assert len(got) >= len(c["exp"]), (c["label"], c["partition"])
        for op, e in zip(got, c["exp"]):
            assert op.Node == e["node"] and op.State == e["state"], (c["label"], c["partition"], got, c["exp"])


# ---- randomised instances: same interned tables through CUDA and through the oracle ---------

@pytest.mark.parametrize("chunk", range(16))
def test_random_instances_gpu_vs_oracle(chunk):
    L = literal()
    for seed in range(chunk * 60, (chunk + 1) * 60):
        kw = random_instance(seed)
        ip = _host.intern_plan(**copy.deepcopy(kw))
        ref = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, ref.out_ptr) == 0
        got = _host.plan_out(ip)
        _host.run_plan_cuda(ip, got)
        assert np.array_equal(got.next_rows, ref.next_rows), seed
        assert np.array_equal(got.next_shape, ref.next_shape), seed
        assert np.array_equal(got.warn, ref.warn), seed
        assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps), seed
        if seed % 10 == 0:   # and the whole string round trip against the literal oracle
            lit = L.plan_next_map_ex(**copy.deepcopy(kw))
            r = _host.PlanNextMapEx(**copy.deepcopy(kw))
            assert r["next_map"] == lit["next_map"] and r["warnings"] == lit["warnings"], seed


def random_tables(seed):
    """Mid-size random flat instances (hundreds to thousands of partitions): large enough for the sequencer
    kernel to be picked, with churn, weights, stickiness, partial assignment and nodes outside nodesAll."""
    rng = np.random.default_rng(seed)
    N = int(rng.integers(6, 160))
    S = int(rng.integers(1, 4))
    k = [int(rng.integers(1, 4)) if s < 2 else int(rng.integers(0, 2)) for s in range(S)]
    if np.random.default_rng([seed, 4]).random() < 0.25:   # k = 4 from a stream of its own: other seeds keep their instances
        k[0] = 4
    while sum(k) > N - 2:
        k = [max(1, x - 1) if s == 0 else max(0, x - 1) for s, x in enumerate(k)]
    P = int(rng.integers(70, 2500))
    NU = N + int(rng.integers(0, 3))
    t = tables.PlanTables(N, S, P, list(range(S)), k, n_node_ids=NU)
    SL = t.n_slots
    rows = np.full((P, SL), -1, np.int32)
    live = max(SL + 1, N - int(rng.integers(0, 4)))
    for p in range(P):
        perm = rng.permutation(live)[:SL]
        for s in range(S):
            lo, hi = int(t.state_slot_off[s]), int(t.state_slot_off[s + 1])
            n = hi - lo if rng.random() < 0.9 else int(rng.integers(0, hi - lo + 1))
            rows[p, lo:lo + n] = perm[lo:lo + n]
    if NU > N and P > 3:
        rows[1, SL - 1] = N            # a node name that is not in nodesAll
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    if rng.random() < 0.3:             # partitionsToAssign differs from prevMap for some rows
        sel = rng.random(P) < 0.05
        t.cur_rows[sel] = -1
    sh = (np.ones((P, S)) * 2).astype(np.uint8)
    t.prev_shape[:] = sh
    t.cur_shape[:] = sh
    t.part_in_prev[:] = 1
    if rng.random() < 0.3:
        t.part_in_assign[:] = (rng.random(P) < 0.8).astype(np.uint8)
    n_rm = int(rng.integers(0, max(1, N // 8)))
    t.node_removed[rng.permutation(N)[:n_rm]] = 1
    t.node_added[rng.permutation(N)[:int(rng.integers(0, N // 4 + 1))]] = 1
    t.add_is_nil = int(rng.random() < 0.1)
    if rng.random() < 0.6:
        t.has_node_weights = 1
        t.node_has_weight[:] = (rng.random(N) < 0.8).astype(np.uint8)
        t.node_weight[:] = rng.integers(-2, 7, N)
        t.booster_kind = int(rng.random() < 0.5)
    if rng.random() < 0.6:
        t.has_part_weights = 1
        t.part_has_weight[:] = (rng.random(P) < 0.4).astype(np.uint8)
        t.part_weight[:] = rng.integers(1, 9, P)
        t.state_has_stickiness[:] = (rng.random(S) < 0.7).astype(np.uint8)
        t.state_stickiness[:] = rng.integers(0, 5, S)
    t.max_iters = int(rng.integers(1, 6))
    return t


@pytest.mark.parametrize("chunk", range(6))
def test_random_midsize_tables_gpu_vs_oracle(ctx, chunk):
    for seed in range(chunk * 8, (chunk + 1) * 8):
        t = random_tables(seed)
        ref = oracle_tables(t)
        for engine in (0, 1, 2):
            t.engine = engine
            got = ctx.plan_next_map(t)
            assert np.array_equal(got.next_rows, ref.next_rows), (seed, engine)
            assert np.array_equal(got.next_shape, ref.next_shape) and np.array_equal(got.warn, ref.warn), (seed, engine)
            assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps), (seed, engine)


def test_all_nodes_removed_gives_nil_lists(ctx):
    # candidateNodes stays a nil slice when nodesNext is empty (plan.go:142): shape NIL, 10 iterations
    L = literal()
    # (with a second state the later pass turns the list into a non-nil empty one, misc.go:29)
    kw = dict(prev_map={"0": {}, "1": {}}, partitions_to_assign=None, nodes_all=["a", "b"], nodes_to_remove=["a", "b"],
              nodes_to_add=[], model={"primary": (0, 1)})
    lit = L.plan_next_map_ex(**copy.deepcopy(kw))
    r = _host.PlanNextMapEx(**kw)
    assert r["next_map"] == lit["next_map"]
    assert r["next_map"]["0"]["primary"] is None
    assert r["warnings"] == lit["warnings"] and r["iterations"] == lit["iterations"]


# ---- BASELINE.json configurations ---------------------------------------------------------------

def two_stage(ctx, cfg, P=None, engine=0):
    """fresh placement, then the configuration's rebalance; engine 0 = auto (the sequencer kernel takes the
    sticky passes), 1 = lock-step kernel only.  Both must equal the oracle bit for bit."""
    fresh = synth.make_fresh(cfg, P=P)
    fresh.engine = engine
    ref1 = oracle_tables(fresh)
    got1 = ctx.plan_next_map(fresh)
    assert_same(got1, ref1)
    if cfg == 1:
        return got1
    reb = synth.make_rebalance(cfg, None if cfg == 4 else got1.next_rows, P=P)
    reb.engine = engine
    ref2 = oracle_tables(reb)
    got2 = ctx.plan_next_map(reb)
    assert_same(got2, ref2)
    return got2


@pytest.mark.parametrize("N", [1500, 3000, 6000])
def test_many_nodes_every_engine(ctx, N):
    """Clusters with more than 1 024 nodes (4, 8 and 16 nodes per thread in the lock-step / sequencer kernels, the team
    evaluation of the speculative kernel up to 2 048): rebalance with weights and stickiness, every engine against the
    oracle."""
    t = synth.make_rebalance(4, P=6144, N=N)
    ref = oracle_tables(t)
    for engine in (0, 1, 2):
        t.engine = engine
        assert_same(ctx.plan_next_map(t), ref)


def test_cfg1_64x8(ctx):
    two_stage(ctx, 1)


def test_cfg2_4096x64_rack_rules(ctx):
    two_stage(ctx, 2)


def test_cfg3_65536x256_three_states_zone_rack(ctx):
    two_stage(ctx, 3)


def test_cfg4_weights_stickiness_reduced(ctx):
    two_stage(ctx, 4, P=32768)


@pytest.mark.parametrize("cfg,P", [(2, None), (3, 8192), (4, 16384)])
def test_lockstep_engine_only(ctx, cfg, P):
    two_stage(ctx, cfg, P=P, engine=1)


def test_sequencer_odd_shapes(ctx):
    """k = 3 (10 steps per window), a 4th state with k = 0 and nodes that are not a power of two."""
    t = synth.PlanTables(200, 3, 6000, [0, 1, 2], [1, 3, 0])
    rng = np.random.default_rng(5)
    rows = np.stack([rng.permutation(180)[:4] for _ in range(t.n_parts)]).astype(np.int32)
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    t.prev_shape[:, :2] = 2
    t.cur_shape[:, :2] = 2
    t.part_in_prev[:] = 1
    t.node_removed[:5] = 1
    t.node_added[180:] = 1
    t.has_node_weights = 1
    t.node_has_weight[:] = 1
    t.node_weight[:] = rng.integers(1, 6, t.n_nodes)
    assert_same(ctx.plan_next_map(t), oracle_tables(t))


def test_cfg4_full_size_properties(ctx):
    """1 048 576 x 1 024 through the C ABI with host buffers; checked by size-independent
    properties: every row has its k distinct live nodes, nothing stays on a removed node,
    weighted node loads are conserved.  (The headline cluster does not converge - the
    reference's loop runs all 10 iterations - so there is no fixed point to re-plan; the
    bit-exact check of the same plan is test_cfg4_full_size_bit_exact.)"""
    t = synth.make_rebalance(4)
    r = ctx.plan_next_map(t)
    rows = r.next_rows
    assert (rows >= 0).all() and (rows < t.n_nodes).all()
    assert not np.isin(rows, np.nonzero(t.node_removed)[0]).any()
    srt = np.sort(rows, axis=1)
    assert (srt[:, 1:] != srt[:, :-1]).all()                 # primary and both replicas distinct
    assert r.warn.sum() == 0
    assert r.iters_run == 10 and r.converged == 0 and r.steps == 20 * t.n_parts
    w = np.where(t.part_has_weight > 0, t.part_weight, 1).astype(np.int64)
    assert np.bincount(rows.reshape(-1), np.repeat(w, rows.shape[1]), t.n_nodes).sum() == w.sum() * rows.shape[1]


def test_cfg4_full_size_bit_exact(ctx):
    """THE headline workload (BASELINE.json configs[3]: 1 048 576 partitions x 1 024 nodes, node and
    partition weights, stickiness, -16/+16 nodes; all 10 iterations of plan.go:32-56, 20 findBestNodes
    steps per partition) through blance_plan_next_map AND through the array-form CPU oracle
    (oracle/fast.c, ~2 minutes on one host core): rows, shapes, warnings, iteration and step counts
    must be identical.  Stickiness with PartitionWeights != nil (plan.go:104-115) is pinned here -
    no reference golden covers it."""
    t = synth.make_rebalance(4)
    got = ctx.plan_next_map(t)
    ref = oracle_tables(t)
    assert_same(got, ref)


def test_cfg4_full_size_fresh_bit_exact(ctx):
    """The full-size FRESH placement of cfg 4 (empty previous map: every step is an N-way arg-min with
    massive score ties, the worst case for the (score, position) order), two convergence iterations,
    GPU against the array-form oracle."""
    t = synth.make_fresh(4)
    t.max_iters = 2
    got = ctx.plan_next_map(t)
    ref = oracle_tables(t)
    assert_same(got, ref)


def test_batch_equals_individual(ctx):
    ts, refs = [], []
    for i in range(24):
        f = synth.make_fresh(5, seed_offset=i, P=128 + 8 * i)
        ts.append(f)
        refs.append(oracle_tables(f))
    got = ctx.plan_next_map_batch(ts)
    for g, r in zip(got, refs):
        assert_same(g, r)
    # rebalance stage, different shapes in one batch (cfg 2-style and weighted flat instances)
    ts2 = [synth.make_rebalance(5, g.next_rows, seed_offset=i, P=128 + 8 * i) for i, g in enumerate(got)]
    ts2.append(synth.make_rebalance(4, P=300, N=96))
    refs2 = [oracle_tables(t) for t in ts2]
    for g, r in zip(ctx.plan_next_map_batch(ts2), refs2):
        assert_same(g, r)


def test_wide_batch_every_instance_vs_oracle(ctx):
    """160 instances in one batch: more CTAs than half the SMs, so the pass kernels run in their narrow
    configuration (4 scouts per CTA / one sequencer warp) - the path BASELINE config 5 takes.  Every instance is
    compared with the oracle, for the default engine and for round 1's sequencer kernel."""
    fresh = [synth.make_fresh(5, seed_offset=i, P=96 + 4 * (i % 40)) for i in range(160)]
    got = ctx.plan_next_map_batch(fresh)
    for g, t in zip(got, fresh):
        assert_same(g, oracle_tables(t))
    for engine in (0, 2):
        rebs = [synth.make_rebalance(5, g.next_rows, seed_offset=i, P=96 + 4 * (i % 40)) for i, g in enumerate(got)]
        for t in rebs:
            t.engine = engine
        for g, t in zip(ctx.plan_next_map_batch(rebs), rebs):
            assert_same(g, oracle_tables(t))


def test_multi_device_context_shards_a_batch():
    """blance_ctx_create_multi: the batch is spread over every visible GPU (instance i -> device i mod G); results
    must not depend on where an instance ran.  With one visible GPU this still exercises the dispatch code."""
    import torch
    G = max(1, min(8, torch.cuda.device_count()))
    mctx = tables.Context(device_ids=list(range(G)))
    assert mctx.device_count() == G
    ts = [synth.make_rebalance(4, P=512 + 64 * i, N=96) for i in range(2 * G + 1)]
    for g, t in zip(mctx.plan_next_map_batch(ts), ts):
        assert_same(g, oracle_tables(t))
    # single-plan entry points of a multi-device context run on its first device
    assert_same(mctx.plan_next_map(ts[0]), oracle_tables(ts[0]))
    mctx.close()


def test_resident_plan_replay(ctx):
    t = synth.make_rebalance(4, P=4096)
    ref = oracle_tables(t)
    plan = ctx.upload(t)
    for _ in range(2):
        ctx.run(plan)
        assert_same(ctx.fetch(plan, tables.PlanResult(t)), ref)
    ctx.free(plan)


# ---- CalcPartitionMoves as a vectorised map diff ------------------------------------------------------

def test_calc_partition_moves_vectorised(ctx):
    rng = np.random.default_rng(7)
    for favor in (0, 1):
        for S, caps in ((2, (1, 2)), (3, (1, 2, 1)), (3, (2, 2, 2))):
            slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
            P, SL = 5000, int(slot_off[-1])
            def rows():
                r = np.full((P, SL), -1, np.int32)
                for p in range(P):
                    perm = rng.permutation(8)[:SL]
                    for s in range(S):
                        n = rng.integers(0, caps[s] + 1)
                        r[p, slot_off[s]:slot_off[s] + n] = perm[slot_off[s]:slot_off[s] + n]
                return r
            beg, end = rows(), rows()
            got = ctx.calc_partition_moves(slot_off, beg, end, favor)
            max_ops = 2 * SL
            on = np.zeros((P, max_ops), np.int32); os_ = np.zeros((P, max_ops), np.uint8)
            ok = np.zeros((P, max_ops), np.uint8); oc = np.zeros(P, np.int32)
            assert FAST.oracle_fast_calc_partition_moves(P, S, S, slot_off.ctypes.data, beg.ctypes.data, end.ctypes.data,
                                                         favor, max_ops, on.ctypes.data, os_.ctypes.data, ok.ctypes.data,
                                                         oc.ctypes.data) == 0
            assert np.array_equal(got[3], oc)
            m = np.arange(max_ops)[None, :] < oc[:, None]
            assert np.array_equal(got[0][m], on[m]) and np.array_equal(got[1][m], os_[m]) and np.array_equal(got[2][m], ok[m])


def test_moves_plan_csr_and_available_moves(ctx):
    """blance_moves_*: the orchestrator's seeding (orchestrate.go:273-287) as device-resident CSR move lists, one
    round of findAvailableMovesUnlocked (orchestrate.go:749-763) for random cursors and the lowest-MoveOpWeight pick
    per node (orchestrate.go:177-186), against the oracle restatement."""
    FAST.oracle_fast_moves_available.argtypes = [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 7
    rng = np.random.default_rng(11)
    for favor, caps, NN in ((0, (1, 2), 40), (1, (1, 2, 1), 12), (0, (2, 2, 2), 9)):
        S = len(caps)
        slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
        P, SL = 20000, int(slot_off[-1])

        def rows():
            r = np.full((P, SL), -1, np.int32)
            for p in range(P):
                perm = rng.permutation(NN)[:SL]
                for s_ in range(S):
                    n = rng.integers(0, caps[s_] + 1)
                    r[p, slot_off[s_]:slot_off[s_] + n] = perm[slot_off[s_]:slot_off[s_] + n]
            return r
        beg, end = rows(), rows()
        max_ops = 2 * SL
        on = np.zeros((P, max_ops), np.int32); os_ = np.zeros((P, max_ops), np.uint8)
        ok = np.zeros((P, max_ops), np.uint8); oc = np.zeros(P, np.int32)
        assert FAST.oracle_fast_calc_partition_moves(P, S, S, slot_off.ctypes.data, beg.ctypes.data, end.ctypes.data, favor, max_ops,
                                                     on.ctypes.data, os_.ctypes.data, ok.ctypes.data, oc.ctypes.data) == 0
        h, total = ctx.moves_create(slot_off, beg, end, favor, NN)
        off, node, state, kind = ctx.moves_fetch(h, total)
        ref_off = np.concatenate([[0], np.cumsum(oc)]).astype(np.int64)
        assert total == int(oc.sum()) and np.array_equal(off, ref_off)
        m = np.arange(max_ops)[None, :] < oc[:, None]
        assert np.array_equal(node, on[m]) and np.array_equal(state, os_[m]) and np.array_equal(kind, ok[m])
        for rnd in range(3):
            nxt = rng.integers(0, max_ops + 1, P).astype(np.int32) if rnd else np.zeros(P, np.int32)
            node_off, node_parts, best = ctx.moves_available(h, nxt)
            r_off = np.zeros(NN + 1, np.int32); r_parts = np.zeros(P, np.int32); r_best = np.zeros(NN, np.int32)
            assert FAST.oracle_fast_moves_available(P, NN, ref_off.ctypes.data, node.ctypes.data, kind.ctypes.data, nxt.ctypes.data,
                                                    r_off.ctypes.data, r_parts.ctypes.data, r_best.ctypes.data) == 0
            assert np.array_equal(node_off, r_off) and np.array_equal(node_parts, r_parts[:r_off[-1]]) and np.array_equal(best, r_best)
        ctx.moves_free(h)


def test_invalid_arguments_are_status_codes(ctx):
    t = synth.make_fresh(1)
    t.top_state = 7
    with pytest.raises(blance_b200.BlanceError):
        ctx.plan_next_map(t)
    t = synth.make_fresh(1)
    t.state_constraints = np.array([40, 1], np.int32)        # > 16: unsupported, reported, not silently clipped
    with pytest.raises(blance_b200.BlanceError):
        ctx.plan_next_map(t)
