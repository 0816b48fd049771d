"""blance_moves_exposure on the device: equal, field for field, to the literal replay on random move lists (with and
without a fault-domain forest), to the vectorised oracle on the synthetic configurations and on the full-size
headline rebalance, consistent with blance_map_audit at both ends, and the edges.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import exposure_oracle as EO
from test_exposure_oracle import random_case, random_forest
from test_schedule_gpu import _plan_moves

from blance_b200 import synth, tables
from blance_b200.abi import BlanceError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def device_and(ctx, oracle, slot_off, beg, h, total, c, cons, top, NN, parent=None, mover=None):
    """Schedules handle h at count c, runs the exposure and the oracle on the fetched tables; asserts equality."""
    ro, so, sc = ctx.moves_schedule(h, c, mover)
    got = ctx.moves_exposure(h, cons, top, parent)
    off, node, state, kind = ctx.moves_fetch(h, total)
    want = oracle(slot_off, beg, off, node, state, kind, ro, so, cons, top, NN, parent)
    EO.assert_equal(got, want, (c, top))
    return got, sc


def test_random_lists_equal_the_literal_replay(ctx):
    rng = np.random.default_rng(41)
    for trial in range(40):
        slot_off, beg, end, cons, top, NN = random_case(rng)
        h, total = ctx.moves_create(slot_off, beg, end, trial % 2 == 0, NN, n_visit_states=None if trial % 3 else 1)
        mover = (rng.random(NN) >= 0.15).astype(np.uint8) if trial % 4 == 1 else None
        parent = random_forest(rng, NN, int(rng.integers(0, 17))) if trial % 2 else None
        for c in (1, 2, 4):
            device_and(ctx, EO.replay, slot_off, beg, h, total, c, cons, top, NN, parent, mover)
        ctx.moves_free(h)


def test_larger_random_lists_equal_the_vectorised_oracle(ctx):
    rng = np.random.default_rng(42)
    for trial in range(6):
        slot_off, beg, end, cons, top, NN = random_case(rng, P=20000, NN=int(rng.integers(8, 300)))
        h, total = ctx.moves_create(slot_off, beg, end, trial % 2 == 0, NN)
        parent = random_forest(rng, NN, 16) if trial % 2 else None
        for c in (1, 4):
            device_and(ctx, EO.vectorised, slot_off, beg, h, total, c, cons, top, NN, parent)
        ctx.moves_free(h)


@pytest.mark.parametrize("cfg,P", [(1, None), (2, None), (3, 8192), (4, 32768)])
def test_synthetic_configurations(ctx, cfg, P):
    t, prev, nxt = _plan_moves(ctx, cfg, P)
    cons = np.asarray(t.state_constraints, np.int32)
    for favor in (False, True):
        h, total = ctx.moves_create(t.state_slot_off, prev, nxt, favor, t.n_node_ids)
        for c in (1, 2, 4):
            got, sc = device_and(ctx, EO.vectorised, t.state_slot_off, prev, h, total, c, cons, t.top_state, t.n_node_ids)
            # the ends against the audit of the beg and end maps (every partition lists every constrained state)
            audits = [ctx.map_audit(t, rows, np.full((t.n_parts, t.n_states), 2, np.uint8)) for rows in (prev, nxt)]
            for k, a in ((0, audits[0]), (got["rounds"], audits[1])):
                if k and sc["stuck_parts"]:
                    continue
                assert got["series"][EO.METRICS.index("SHORT"), k] == a.short_parts
                assert got["series"][EO.METRICS.index("NO_TOP"), k] == a.no_top_parts
            for a in audits:
                assert (got["dom_peak"] >= a.dom_all).all()
        ctx.moves_free(h)


def test_full_size_headline_rebalance(ctx):
    t = synth.make_rebalance(4)
    nxt = ctx.plan_next_map(t).next_rows
    cons = np.asarray(t.state_constraints, np.int32)
    h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, nxt, False, t.n_node_ids)
    for c in (1, 2, 4):
        got, sc = device_and(ctx, EO.vectorised, t.state_slot_off, t.prev_rows, h, total, c, cons, t.top_state, t.n_node_ids)
        assert sc["stuck_parts"] == 0 and got["rounds"] == sc["rounds"] > 0
    ctx.moves_free(h)


def test_edges(ctx):
    rng = np.random.default_rng(5)
    slot_off, beg, end, cons, top, NN = random_case(rng, P=300, NN=6)
    h, total = ctx.moves_create(slot_off, beg, end, True, NN)
    with pytest.raises(BlanceError, match="no schedule"):
        ctx.moves_exposure(h, cons, top)
    # a second schedule with another count: the exposure follows it
    for c in (1, 3):
        device_and(ctx, EO.replay, slot_off, beg, h, total, c, cons, top, NN)
    # no top state
    device_and(ctx, EO.replay, slot_off, beg, h, total, 2, cons, -1, NN)
    # argument errors
    for bad_cons, bad_top, match in ((np.full(len(cons), -1), top, "negative"), (cons, len(cons), "top_state")):
        with pytest.raises(BlanceError, match=match):
            ctx.moves_exposure(h, bad_cons, bad_top)
    with pytest.raises(BlanceError, match="domain_parent"):
        ctx.moves_exposure(h, cons, top, np.full(NN, NN + 5, np.int32))
    ctx.moves_free(h)
    # zero ops (no entries on either side), zero partitions
    blank = np.full_like(beg, -1)
    h, total = ctx.moves_create(slot_off, blank, blank, False, NN)
    got, sc = device_and(ctx, EO.replay, slot_off, blank, h, total, 1, cons, top, NN)
    assert total == 0 and got["rounds"] == 0 and got["series"].shape == (6, 1)
    ctx.moves_free(h)
    empty = np.zeros((0, int(slot_off[-1])), np.int32)
    h, total = ctx.moves_create(slot_off, empty, empty, False, NN)
    device_and(ctx, EO.replay, slot_off, empty, h, total, 1, cons, top, NN)
    ctx.moves_free(h)


# (seed, P, node ids, count) -> kernels blance_moves_schedule launches, counted with the library as it was before
# blance_moves_exposure existed; the schedule's launch sequence follows its rounds, so these pin it
SCHEDULE_LAUNCHES = {(8, 2000, 12, 2): 1156, (9, 5000, 40, 1): 2116, (10, 300, 6, 4): 196}


@pytest.mark.parametrize("case", sorted(SCHEDULE_LAUNCHES))
def test_schedule_launches_are_unchanged(ctx, case):
    seed, P, NN, c = case
    slot_off, beg, end, cons, top, _ = random_case(np.random.default_rng(seed), P=P, NN=NN)
    h, _ = ctx.moves_create(slot_off, beg, end, False, NN)
    for _ in range(2):                       # before and after an exposure on the handle
        n0 = ctx.kernel_launches()
        ctx.moves_schedule(h, c)
        assert ctx.kernel_launches() - n0 == SCHEDULE_LAUNCHES[case]
        ctx.moves_exposure(h, cons, top)
    ctx.moves_free(h)
