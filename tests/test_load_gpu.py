"""blance_moves_load on the device: equal, field for field, to the literal replay on random move lists (with and
without weights), to the vectorised oracle on the synthetic configurations and on the full-size headline rebalance,
countStateNodes of the beg and end maps at both ends, the argument errors, the load's own launch count, and the
launch counts of the schedule and the exposure unchanged by it.  Needs an H100; run with -m gpu."""
import numpy as np
import pytest

import load_oracle as LO
from exposure_oracle import beg_entries
from test_exposure_gpu import SCHEDULE_LAUNCHES
from test_exposure_oracle import random_case
from test_load_oracle import random_weights
from test_schedule_gpu import _plan_moves

from blance_b200 import synth, tables
from blance_b200.abi import BlanceError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def device_and(ctx, oracle, slot_off, beg, h, total, c, NN, w=None, has=None, mover=None):
    """Schedules handle h at count c, runs the load and the oracle on the fetched tables; asserts equality."""
    ro, so, sc = ctx.moves_schedule(h, c, mover)
    got = ctx.moves_load(h, w, has)
    off, node, state, kind = ctx.moves_fetch(h, total)
    eff = None if w is None else np.where(np.ones(len(w), bool) if has is None else np.asarray(has) != 0, w, 1)
    want = oracle(slot_off, beg, off, node, state, kind, ro, so, NN, eff)
    LO.assert_equal(got, want, c)
    assert got["kernel_ms"] > 0
    return got, sc


def count_state_nodes(slot_off, rows, NU, w):
    """countStateNodes (plan.go:374-399) of a map given as rows, per state and node, and the all-state row."""
    S = len(slot_off) - 1
    out = np.zeros((S + 1, NU), np.int64)
    for s in range(S):
        for x in range(slot_off[s], slot_off[s + 1]):
            live = (rows[:, slot_off[s]:x + 1] != -1).all(axis=1)        # before the state's first empty slot
            np.add.at(out[s], rows[live, x], w[live])
    out[S] = out[:S].sum(axis=0)
    return out


def test_random_lists_equal_the_literal_replay(ctx):
    rng = np.random.default_rng(51)
    for trial in range(40):
        slot_off, beg, end, _, _, NN = random_case(rng)
        h, total = ctx.moves_create(slot_off, beg, end, trial % 2 == 0, NN, n_visit_states=None if trial % 3 else 1)
        mover = (rng.random(NN) >= 0.15).astype(np.uint8) if trial % 4 == 1 else None
        w = random_weights(rng, beg.shape[0], trial % 3)
        has = (rng.random(beg.shape[0]) < 0.7).astype(np.uint8) if w is not None and trial % 2 else None
        for c in (1, 2, 4):
            eff = np.ones(beg.shape[0], np.int64) if w is None else np.where(np.ones(len(w), bool) if has is None else has != 0, w, 1)
            if int(eff.sum()) * max(1, int(slot_off[-1])) >= 1 << 31:     # the load bound
                ctx.moves_schedule(h, c, mover)
                with pytest.raises(BlanceError, match="2\\^31"):
                    ctx.moves_load(h, w, has)
                continue
            device_and(ctx, LO.replay, slot_off, beg, h, total, c, NN, w, has, mover)
        ctx.moves_free(h)


def test_larger_random_lists_equal_the_vectorised_oracle(ctx):
    rng = np.random.default_rng(52)
    for trial in range(6):
        slot_off, beg, end, _, _, NN = random_case(rng, P=20000, NN=int(rng.integers(8, 300)))
        h, total = ctx.moves_create(slot_off, beg, end, trial % 2 == 0, NN)
        w = rng.integers(0, 1000, beg.shape[0]) if trial % 2 else None
        for c in (1, 4):
            device_and(ctx, LO.vectorised, slot_off, beg, h, total, c, NN, w)
        ctx.moves_free(h)


@pytest.mark.parametrize("cfg,P", [(1, None), (2, None), (3, 8192), (4, 32768)])
def test_synthetic_configurations(ctx, cfg, P):
    t, prev, nxt = _plan_moves(ctx, cfg, P)
    w, has = (t.part_weight, t.part_has_weight) if t.has_part_weights else (None, None)
    eff = np.where(t.part_has_weight != 0, t.part_weight, 1).astype(np.int64) if t.has_part_weights else np.ones(t.n_parts, np.int64)
    for favor in (False, True):
        h, total = ctx.moves_create(t.state_slot_off, prev, nxt, favor, t.n_node_ids)
        for c in (1, 2, 4):
            got, sc = device_and(ctx, LO.vectorised, t.state_slot_off, prev, h, total, c, t.n_node_ids, w, has)
            assert np.array_equal(got["node_beg"], count_state_nodes(t.state_slot_off, prev, t.n_node_ids, eff))
            if sc["stuck_parts"] == 0:
                assert np.array_equal(got["node_end"], count_state_nodes(t.state_slot_off, nxt, t.n_node_ids, eff))
        ctx.moves_free(h)


def test_full_size_headline_rebalance(ctx):
    t = synth.make_rebalance(4)
    nxt = ctx.plan_next_map(t).next_rows
    eff = np.where(t.part_has_weight != 0, t.part_weight, 1).astype(np.int64)
    h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, nxt, False, t.n_node_ids)
    for c in (1, 2, 4):
        got, sc = device_and(ctx, LO.vectorised, t.state_slot_off, t.prev_rows, h, total, c, t.n_node_ids,
                             t.part_weight, t.part_has_weight)
        assert sc["stuck_parts"] == 0 and got["rounds"] == sc["rounds"] > 0
        assert np.array_equal(got["node_end"], count_state_nodes(t.state_slot_off, nxt, t.n_node_ids, eff))
    ctx.moves_free(h)


def test_edges(ctx):
    rng = np.random.default_rng(6)
    slot_off, beg, end, _, _, NN = random_case(rng, P=300, NN=6)
    h, total = ctx.moves_create(slot_off, beg, end, False, NN)
    with pytest.raises(BlanceError, match="no schedule"):
        ctx.moves_load(h)
    # a second schedule with another count: the load follows it
    for c in (1, 3):
        device_and(ctx, LO.replay, slot_off, beg, h, total, c, NN)
    # weights: the range, a weight a partition does not have is not read, the bound at 2^31
    P = beg.shape[0]
    for bad in (-1, 1000000000):
        w = np.ones(P, np.int32)
        w[7] = bad
        with pytest.raises(BlanceError, match="partition 7 is outside"):
            ctx.moves_load(h, w)
        has = np.ones(P, np.uint8)
        has[7] = 0
        device_and(ctx, LO.replay, slot_off, beg, h, total, 2, NN, w, has)
    w = np.zeros(P, np.int32)
    SL = int(slot_off[-1])
    w[:3] = ((1 << 31) + SL - 1) // SL // 3 + 1                      # sum x n_slots just reaches 2^31
    assert int(w.sum()) * SL >= 1 << 31 and w.max() <= 999999999
    with pytest.raises(BlanceError, match="2\\^31"):
        ctx.moves_load(h, w)
    w[:3] = ((1 << 31) - 1) // SL // 3                               # just below: exact
    device_and(ctx, LO.replay, slot_off, beg, h, total, 2, NN, w)
    ctx.moves_free(h)
    # zero ops (no entries on either side), zero partitions
    blank = np.full_like(beg, -1)
    h, total = ctx.moves_create(slot_off, blank, blank, False, NN)
    got, _ = device_and(ctx, LO.replay, slot_off, blank, h, total, 1, NN)
    assert total == 0 and got["rounds"] == 0 and not got["node_peak"].any() and got["over_node"] == 0
    ctx.moves_free(h)
    empty = np.zeros((0, SL), np.int32)
    h, total = ctx.moves_create(slot_off, empty, empty, False, NN)
    device_and(ctx, LO.replay, slot_off, empty, h, total, 1, NN)
    ctx.moves_free(h)


def has_events(slot_off, beg, op_off, op_node, op_state, op_kind, sched_op, NN):
    """Whether the load of unit weights has an event: an op scheduled before its partition's first unscheduled one, on
    a node in range, that changes the node's entries of some state."""
    S = len(slot_off) - 1
    done = np.zeros(len(op_node), bool)
    done[np.asarray(sched_op, np.int64)] = True
    for p in range(len(op_off) - 1):
        live = beg_entries(slot_off, beg[p])
        for k in range(op_off[p], op_off[p + 1]):
            if not done[k]:
                break
            n = int(op_node[k])
            before = [live.count((n, s)) for s in range(S)]
            live = [e for e in live if e[0] != n]
            after = [int(op_kind[k] != LO.DEL and s == op_state[k]) for s in range(S)]
            if 0 <= n < NN and before != after:
                return True
    return False


@pytest.mark.parametrize("case", sorted(SCHEDULE_LAUNCHES))
def test_schedule_and_exposure_launches_are_unchanged(ctx, case):
    seed, P, NN, c = case
    slot_off, beg, end, cons, top, _ = random_case(np.random.default_rng(seed), P=P, NN=NN)
    h, total = ctx.moves_create(slot_off, beg, end, False, NN)
    expo, load = [], []
    for _ in range(2):                       # before and after a load on the handle
        n0 = ctx.kernel_launches()
        _, so, sc = ctx.moves_schedule(h, c)
        assert ctx.kernel_launches() - n0 == SCHEDULE_LAUNCHES[case]
        n0 = ctx.kernel_launches()
        ctx.moves_exposure(h, cons, top)
        expo.append(ctx.kernel_launches() - n0)
        n0 = ctx.kernel_launches()
        ctx.moves_load(h)
        load.append(ctx.kernel_launches() - n0)
    assert expo[0] == expo[1]
    # the load's own kernels (CUB's are not counted): the op rounds when the schedule moved anything, walk<0> over the
    # partitions, init and final over the (state, node) keys, walk<1> when there are events and peak when there are
    # merged runs, which every event starts or joins
    M = sc["moves_done"]
    ev = has_events(slot_off, beg, *ctx.moves_fetch(h, total), so[:M], NN)
    want = (M > 0) + (P > 0) + (len(slot_off) * NN > 0) * (2 + 2 * ev)
    assert ev and load == [want, want], (ev, load, want)
    ctx.moves_free(h)
