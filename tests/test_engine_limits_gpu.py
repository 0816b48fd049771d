"""The three pass kernels at the limits where `k_pick_mode` (aux_kernels.cuh) switches between them: the
speculative kernel (auto engine; BLANCE_NO_SEQ keeps the sequencer out), the sequencer kernel (engine 2) and the
lock-step kernel (engine 1).  Every case plans against the array-form CPU oracle on the same tables (rows,
shapes, warnings, iterations, convergence, steps) AND checks which kernel ran: `sticky_steps` counts the steps the
speculative or sequencer kernel decided without a full evaluation, so it is > 0 when one of them ran and 0 when
only the lock-step kernel did.  The limits:
  - constraint k <= 4 and padded slots SLP <= 8 for both sticky kernels (BL_K_MAX = 16, BL_SLP_MAX = 32 beyond);
  - N <= 2048 for the speculative kernel, <= 768 in a batch wider than sm_count / 2, N <= 4096 and at most 8 nodes
    per thread for the sequencer; pass_shape's node-per-thread steps at 512, 1024, 2048 and 4096 nodes;
  - n_assign >= 64, at least 25 % eligible rows (exactly k clean current nodes), at least 63/64 clean rows (the
    speculative kernel);
  - hierarchy rules x constraints <= 32 picks per step.
Needs an H100; run with `-m gpu`."""
import ctypes

import numpy as np
import pytest

from oracle_loader import fast_lib_path
from test_scenario_options_gpu import assert_scenario, reference_summary

from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu

FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]

SPEC, SEQ, LOCK = "spec", "seq", "lock"


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle_tables(t):
    r = tables.PlanResult(t)
    s = t.struct()
    assert FAST.oracle_fast_plan_next_map(ctypes.byref(s), ctypes.byref(r.out)) == 0
    return r


def assert_same(got, ref, what):
    assert np.array_equal(got.next_rows, ref.next_rows), what
    assert np.array_equal(got.next_shape, ref.next_shape), what
    assert np.array_equal(got.warn, ref.warn), what
    assert (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps), what


def assert_kernel(got, kernel, what):
    if kernel == LOCK:
        assert got.sticky_steps == 0, (what, got.sticky_steps)
    else:
        assert got.sticky_steps > 0, what


def set_engine(monkeypatch, t, kernel):
    """Engine and environment that let only `kernel` (or the lock-step kernel, where it is not eligible) run."""
    t.engine = {SPEC: 0, SEQ: 2, LOCK: 1}[kernel]
    if kernel == SPEC:
        monkeypatch.setenv("BLANCE_NO_SEQ", "1")
    else:
        monkeypatch.delenv("BLANCE_NO_SEQ", raising=False)


def plan_as(ctx, monkeypatch, t, kernel, ran, ref=None, what=""):
    """Plans t with `kernel` allowed, checks it against the oracle and that `ran` is the kernel that ran."""
    ref = ref if ref is not None else oracle_tables(t)
    set_engine(monkeypatch, t, kernel)
    got = ctx.plan_next_map(t)
    assert_same(got, ref, (what, kernel))
    assert_kernel(got, ran, (what, kernel))
    return got


def cluster(N, P, ks, n_rm=2, n_add=2, seed=0, fresh=False, widths=None):
    """A rebalance of a round-robin previous map: every row holds sum(ks) distinct nodes of the first N - n_add
    (slot j of partition p holds node (p + j * stride) mod (N - n_add)), the first n_rm nodes are removed and the
    last n_add added; node weights 1-4, a quarter of the partitions weighted 1-8, stickiness 3 / 2.  Nearly every
    row is clean and holds its k current nodes, so both sticky kernels are eligible.  `fresh`: the same cluster
    from an empty previous map.  `widths`: every state's slot range at least that wide (tables.widen_layout)."""
    S = len(ks)
    t = tables.PlanTables(N, S, P, list(range(S)), ks)
    rng = np.random.default_rng(seed)
    n0 = N - n_add
    if fresh:
        t.node_added[:] = 1
    else:
        stride = max(1, n0 // (t.n_slots + 1))
        rows = ((np.arange(P)[:, None] + stride * np.arange(t.n_slots)[None, :]) % n0).astype(np.int32)
        t.prev_rows[:] = rows
        t.cur_rows[:] = rows
        t.prev_shape[:] = tables.SHAPE_LIST
        t.cur_shape[:] = tables.SHAPE_LIST
        t.part_in_prev[:] = 1
        t.node_removed[:n_rm] = 1
        t.node_added[n0:] = 1
    t.has_node_weights = 1
    t.node_has_weight[:] = 1
    t.node_weight[:] = rng.integers(1, 5, N)
    t.has_part_weights = 1
    t.part_has_weight[:] = rng.random(P) < 0.25
    t.part_weight[:] = np.where(t.part_has_weight > 0, rng.integers(1, 9, P), 1)
    t.state_has_stickiness[:] = 1
    t.state_stickiness[:] = ([3, 2] + [2] * S)[:S]
    return tables.widen_layout(t, widths) if widths is not None else t


# ---- constraint x layout, every kernel ------------------------------------------------------------------------

LAYOUTS = ([([k], None) for k in (1, 2, 3, 4)] +                       # SLP 4
           [([1, 4], None), ([2, 4], None), ([4, 4], None)] +          # SLP 8
           [([k], [k + 2]) for k in (1, 2, 3, 4)])                      # slot range wider than k


@pytest.mark.parametrize("ks,widths", LAYOUTS, ids=lambda v: "x".join(map(str, v)) if v else "tight")
@pytest.mark.parametrize("fresh", [False, True], ids=["rebalance", "fresh"])
def test_constraints_and_layouts_every_kernel(ctx, monkeypatch, ks, widths, fresh):
    t = cluster(256, 4096, ks, fresh=fresh, widths=widths)
    assert t.n_slots <= 8
    ref = oracle_tables(t)
    for kernel in (SPEC, SEQ, LOCK):
        plan_as(ctx, monkeypatch, t, kernel, kernel, ref)


def test_design_section_8_constraints_of_4(ctx, monkeypatch):
    """The 16 384-partition cfg-4 rebalance with its replica constraint raised to 4 (2 current replicas, 4 slots):
    where the speculative kernel's outcome byte once lost node 3's rank."""
    t = tables.scenario_tables(tables.widen_layout(synth.make_rebalance(4, P=16384), [1, 4]), {},
                               dict(state_constraints=np.array([1, 4], np.int32)))
    ref = oracle_tables(t)
    for kernel in (SPEC, SEQ, LOCK):
        plan_as(ctx, monkeypatch, t, kernel, kernel, ref)


def test_constraints_of_4_repeat_on_one_context(ctx, monkeypatch):
    """The speculative kernel's K = 4 plan twice on one context: the same result both times."""
    t = cluster(512, 8192, [4], seed=3)
    ref = oracle_tables(t)
    a = plan_as(ctx, monkeypatch, t, SPEC, SPEC, ref, "first")
    b = plan_as(ctx, monkeypatch, t, SPEC, SPEC, ref, "second")
    assert_same(a, b, "repeat")


# ---- beyond the sticky kernels: only the lock-step kernel may run ---------------------------------------------

def hier_cluster(N, P, k, rules):
    """cluster() with one state and `rules` (include, exclude levels) on it, in a tree of racks of 8 in rows of 8."""
    t = cluster(N, P, [k])
    t.has_hier_rules = 1
    t.rule_off, mask = synth.hierarchy_masks(N, (8, 8), {0: rules}, 1)
    t.n_rules = mask.shape[0]
    t.ie_mask = mask.reshape(-1)
    t.n_hier_bits = N
    return t


BEYOND = {
    "1x4x4_slp12": lambda: cluster(64, 4096, [1, 4, 4]),
    "k5": lambda: cluster(64, 4096, [5]),
    "k8": lambda: cluster(64, 4096, [8]),
    "k16": lambda: cluster(64, 2048, [16]),
    "16x16_sl32": lambda: cluster(64, 2048, [16, 16]),
    "rules4xk8_32_picks": lambda: hier_cluster(256, 2048, 8, [(2, 1), (1, 0), (2, 0), (2, 1)]),
}


@pytest.mark.parametrize("name", list(BEYOND))
def test_beyond_the_sticky_kernels_every_engine_runs_lockstep(ctx, monkeypatch, name):
    t = BEYOND[name]()
    ref = oracle_tables(t)
    for kernel in (SPEC, SEQ, LOCK):
        plan_as(ctx, monkeypatch, t, kernel, LOCK, ref, name)


# ---- node counts ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,ran", [(2048, SPEC), (2049, LOCK)])
def test_speculative_node_limit_single_plan(ctx, monkeypatch, N, ran):
    t = cluster(N, 4096, [2], n_rm=4, n_add=4)
    plan_as(ctx, monkeypatch, t, SPEC, ran, what=N)


@pytest.mark.parametrize("N,ran", [(768, SPEC), (769, LOCK)])
def test_speculative_node_limit_narrow_batch(ctx, monkeypatch, sm_count, N, ran):
    """sm_count // 2 + 1 instances: the 3-scout configuration, whose team covers 32 x 3 x 8 = 768 nodes."""
    ts = [cluster(N, 512 + 8 * i, [2], seed=i) for i in range(sm_count // 2 + 1)]
    monkeypatch.setenv("BLANCE_NO_SEQ", "1")
    for i, (g, t) in enumerate(zip(ctx.plan_next_map_batch(ts), ts)):
        assert_same(g, oracle_tables(t), (N, i))
        assert_kernel(g, ran, (N, i))


@pytest.mark.parametrize("N", [512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192])
def test_node_per_thread_steps_sequencer_and_lockstep(ctx, monkeypatch, N):
    """pass_shape gives 1, 2, 4, 8 and 16 nodes per thread across these counts; above 4096 (16 per thread) the
    sequencer kernel is not allowed."""
    t = cluster(N, 4096, [2], n_rm=4, n_add=4)
    ref = oracle_tables(t)
    plan_as(ctx, monkeypatch, t, SEQ, SEQ if N <= 4096 else LOCK, ref, N)
    plan_as(ctx, monkeypatch, t, LOCK, LOCK, ref, N)
    if N > 4096:
        plan_as(ctx, monkeypatch, t, SPEC, LOCK, ref, N)


# ---- eligibility thresholds (one iteration: one pass, decided on the tables as given) --------------------------

def one_pass(P, k=2, N=128):
    t = cluster(N, P, [k], n_rm=0, n_add=2)
    t.max_iters = 1
    return t


@pytest.mark.parametrize("unclean,ran", [(64, SPEC), (65, LOCK)])
def test_clean_fraction_63_of_64(ctx, monkeypatch, unclean, ran):
    """64 of 4 096 rows unclean leaves exactly 63/64 clean; a node outside nodesAll makes a row unclean."""
    t = one_pass(4096)
    t.n_node_ids = t.n_nodes + 1
    t.node_removed = np.zeros(t.n_node_ids, np.uint8)
    t.node_added = np.append(t.node_added, 0).astype(np.uint8)
    rows = t.cur_rows.copy()
    rows[np.arange(unclean) * 61, 1] = t.n_nodes
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    plan_as(ctx, monkeypatch, t, SPEC, ran, what=unclean)


@pytest.mark.parametrize("P,ran_spec,ran_seq", [(64, SPEC, SEQ), (63, LOCK, LOCK)])
def test_n_assign_64(ctx, monkeypatch, P, ran_spec, ran_seq):
    t = one_pass(P)
    ref = oracle_tables(t)
    plan_as(ctx, monkeypatch, t, SPEC, ran_spec, ref, P)
    plan_as(ctx, monkeypatch, t, SEQ, ran_seq, ref, P)


@pytest.mark.parametrize("eligible,ran_spec,ran_seq", [(1024, SPEC, SEQ), (1023, LOCK, LOCK)])
def test_eligible_fraction_a_quarter(ctx, monkeypatch, eligible, ran_spec, ran_seq):
    """Rows with fewer than k current nodes are clean but not eligible: 1 024 of 4 096 rows keep both nodes."""
    t = one_pass(4096)
    rows = t.cur_rows.copy()
    rows[eligible:, 1] = tables.NO_NODE
    t.prev_rows[:] = rows
    t.cur_rows[:] = rows
    ref = oracle_tables(t)
    plan_as(ctx, monkeypatch, t, SPEC, ran_spec, ref, eligible)
    plan_as(ctx, monkeypatch, t, SEQ, ran_seq, ref, eligible)


# ---- several constraints in one batch -------------------------------------------------------------------------

@pytest.mark.parametrize("width", ["wide", "narrow"])
def test_mixed_constraints_and_engines_in_one_batch(ctx, monkeypatch, sm_count, width):
    """Replica constraints 1-4 and all three engines side by side: one pass launches the speculative and the
    sequencer kernel for several K.  Wide: 2n <= sm_count (9 scouts, 4 sequencer warps); narrow: more than
    sm_count / 2 instances."""
    monkeypatch.delenv("BLANCE_NO_SEQ", raising=False)
    n = 12 if width == "wide" else sm_count // 2 + 1
    assert (2 * n <= sm_count) == (width == "wide")
    ts, ran = [], []
    for i in range(n):
        kernel = (SPEC, SEQ, LOCK)[i % 3]
        t = cluster(256, 1024 + 16 * i, [1, 1 + (i // 3) % 4], seed=i)
        t.engine = {SPEC: 0, SEQ: 2, LOCK: 1}[kernel]
        ts.append(t)
        ran.append(kernel)
    for i, (g, t) in enumerate(zip(ctx.plan_next_map_batch(ts), ts)):
        assert_same(g, oracle_tables(t), i)
        assert_kernel(g, ran[i], i)


# ---- the scenario summary at 32 slots -------------------------------------------------------------------------

def test_scenario_summary_at_32_slots(ctx):
    t = cluster(64, 2048, [16, 16])
    assert t.n_slots == 32
    NU = t.n_node_ids
    scs = []
    for rm in ([], [3], [5, 40]):
        r = t.node_removed.copy()
        r[rm] = 1
        scs.append(dict(node_removed=r, node_added=t.node_added.copy(), add_is_nil=0))
    assert all(len(sc["node_removed"]) == NU for sc in scs)
    res = ctx.plan_scenarios(t, scs, True, want_rows=range(len(scs)))
    for i, (sc, got) in enumerate(zip(scs, res)):
        s = tables.scenario_tables(t, sc)
        ref = oracle_tables(s)
        assert_scenario(got, ref, reference_summary(s, ref.next_rows, ref.warn, True), i)
