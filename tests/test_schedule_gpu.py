"""blance_moves_schedule on the device against the serial oracle (tests/schedule_oracle.c): round_off and sched_op
must be EQUAL, and so must rounds, moves_done, stuck_parts and max_batch.  Random move lists with common weight
ties, the reference's TestOrchestrateConcurrentMoves through blance_b200.OrchestrateSchedule, the move lists of
the synthetic configurations (prev rows -> GPU-planned next rows) including the full-size headline plan, and the
edges.  Needs an H100; run with -m gpu."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import schedule_oracle as SO
from oracle_loader import fast_lib_path
from test_schedule_oracle import COUNTS, check_golden_batch, check_invariants, golden_batch, golden_cases

import blance_b200
from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def schedule_both(ctx, h, total, c, mover=None, NN=None):
    """Device schedule and oracle schedule of handle h's CSR lists; asserts equality, returns the device's."""
    off, node, _, kind = ctx.moves_fetch(h, total)
    ro, so, sc = ctx.moves_schedule(h, c, mover)
    want_ro, want_so, want = SO.schedule(off, node, kind, h[2], c, mover)
    assert np.array_equal(ro, want_ro) and np.array_equal(so, want_so)
    assert {k: sc[k] for k in want} == want
    return off, node, kind, ro, so, sc


def random_rows(rng, P, NN, caps=(1, 2), hot=None):
    slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
    SL = int(slot_off[-1])

    def rows():
        r = np.full((P, SL), -1, np.int32)
        for p in range(P):
            perm = rng.permutation(NN)[:SL]
            if hot is not None and rng.random() < 0.5:
                perm[0] = hot if hot not in perm[1:] else perm[0]
            for s in range(len(caps)):
                n = rng.integers(0, caps[s] + 1)
                r[p, slot_off[s]:slot_off[s] + n] = perm[slot_off[s]:slot_off[s] + n]
        return r
    beg, end = rows(), rows()
    same = rng.random(P) < 0.15                 # partitions without ops
    end[same] = beg[same]
    return slot_off, beg, end


def test_random_lists_equal_the_oracle(ctx):
    rng = np.random.default_rng(21)
    for trial in range(24):
        P, NN = int(rng.integers(1, 3000)), int(rng.integers(2, 40))
        slot_off, beg, end = random_rows(rng, P, NN, hot=0 if trial % 2 else None)
        favor = trial % 3 == 0
        h, total = ctx.moves_create(slot_off, beg, end, favor, NN)
        mover = (rng.random(NN) >= 0.1).astype(np.uint8) if trial % 4 else None
        for c in COUNTS:
            off, node, kind, ro, so, sc = schedule_both(ctx, h, total, c, mover)
            check_invariants(off, node, kind, NN, c, np.ones(NN, np.uint8) if mover is None else mover, ro, so, sc)
        ctx.moves_free(h)


@pytest.mark.parametrize("c", golden_cases(), ids=lambda c: "%d-%s" % (c["index"], c["label"].replace(" ", "_")))
def test_golden_batches_through_orchestrate_schedule(c):
    model = {k: (v["priority"], v["constraints"]) for k, v in c["model"].items()}
    beg = {k: v["nodesByState"] for k, v in c["begMap"].items()}
    end = {k: v["nodesByState"] for k, v in c["endMap"].items()}
    opts = blance_b200.OrchestratorOptions(MaxConcurrentPartitionMovesPerNode=c["maxConcurrentMoves"])
    rounds = blance_b200.OrchestrateSchedule(model, opts, c["nodesAll"], beg, end)
    check_golden_batch(c, golden_batch(c, [[tuple(b) for b in r] for r in rounds]))


def test_orchestrate_schedule_mismatched_maps():
    with pytest.raises(blance_b200.BlanceError, match="mismatched begMap and endMap"):
        blance_b200.OrchestrateSchedule({"primary": (0, 1)}, None, ["a"], {"0": {"primary": ["a"]}}, {})


def _plan_moves(ctx, cfg, P=None):
    fresh = synth.make_fresh(cfg, P=P)
    r1 = ctx.plan_next_map(fresh)
    if cfg == 1:
        return fresh, fresh.prev_rows, r1.next_rows
    reb = synth.make_rebalance(cfg, None if cfg == 4 else r1.next_rows, P=P)
    return reb, reb.prev_rows, ctx.plan_next_map(reb).next_rows


@pytest.mark.parametrize("cfg,P", [(1, None), (2, None), (3, 8192), (4, 32768)])
def test_synthetic_configurations(ctx, cfg, P):
    t, prev, nxt = _plan_moves(ctx, cfg, P)
    for favor in (False, True):
        h, total = ctx.moves_create(t.state_slot_off, prev, nxt, favor, t.n_node_ids)
        assert total > 0
        for c in (1, 2, 4):
            schedule_both(ctx, h, total, c)
        ctx.moves_free(h)


def test_full_size_headline_schedule(ctx):
    """The headline plan (1 048 576 x 1 024, -16/+16 nodes), itself checked against the oracle's digest in
    profiles/parity_cfg4.json, then its move lists scheduled at c = 1 and c = 4 on the device and by the oracle."""
    t = synth.make_rebalance(4)
    r = ctx.plan_next_map(t)
    with open(os.path.join(ROOT, "profiles", "parity_cfg4.json")) as f:
        pj = json.load(f)
    assert pj["n_parts"] == t.n_parts
    assert hashlib.sha256(np.ascontiguousarray(r.next_rows).tobytes()).hexdigest() == pj["sha256_next_rows"]
    assert (r.iters_run, r.steps) == (pj["iters_run"], pj["steps"])
    h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, r.next_rows, False, t.n_node_ids)
    for c in (1, 4):
        _, _, _, ro, so, sc = schedule_both(ctx, h, total, c)
        assert sc["rounds"] > 0 and sc["moves_done"] == total and sc["stuck_parts"] == 0
    ctx.moves_free(h)


def test_edges(ctx):
    rng = np.random.default_rng(3)
    slot_off = np.array([0, 1, 3], np.int32)
    # total_ops == 0
    beg = np.stack([rng.permutation(6)[:3] for _ in range(100)]).astype(np.int32)
    h, total = ctx.moves_create(slot_off, beg, beg, False, 6)
    assert total == 0
    ro, so, sc = ctx.moves_schedule(h, 3)
    assert ro.tolist() == [0] and len(so) == 0 and sc["rounds"] == 0 and sc["stuck_parts"] == 0
    ctx.moves_free(h)
    # n_parts == 0
    h, total = ctx.moves_create(slot_off, np.zeros((0, 3), np.int32), np.zeros((0, 3), np.int32), False, 6)
    ro, so, sc = ctx.moves_schedule(h, 1)
    assert ro.tolist() == [0] and sc["rounds"] == 0
    ctx.moves_free(h)
    # 8 192 node ids
    slot_off, beg, end = random_rows(rng, 20000, 8192)
    h, total = ctx.moves_create(slot_off, beg, end, False, 8192)
    for c in (1, 3):
        schedule_both(ctx, h, total, c)
    ctx.moves_free(h)
    # one node with 12 000 available entries in the first round
    P = 12000
    beg = np.full((P, 3), -1, np.int32)
    beg[:, 0] = 1 + np.arange(P) % 40
    end = np.full((P, 3), -1, np.int32)
    end[:, 0] = 0
    end[::3, 1] = 1 + (np.arange(0, P, 3) + 7) % 40
    h, total = ctx.moves_create(slot_off, beg, end, False, 41)
    for c in (1, 64):
        _, node, _, ro, so, sc = schedule_both(ctx, h, total, c)
        assert sc["max_batch"] == c
    # every node without a mover: nothing runs, every partition with ops is stuck
    ro, so, sc = ctx.moves_schedule(h, 2, np.zeros(41, np.uint8))
    assert sc["rounds"] == 0 and sc["moves_done"] == 0 and sc["stuck_parts"] == P and ro.tolist() == [0]
    ctx.moves_free(h)
    # 320 ops per partition: 160 slots per row, every node changing
    perms = np.stack([rng.permutation(320) for _ in range(3)]).astype(np.int32)
    h, total = ctx.moves_create(np.array([0, 160], np.int32), perms[:, :160], perms[:, 160:], False, 320)
    for c in (1, 4):
        off, _, _, _, _, _ = schedule_both(ctx, h, total, c)
        assert np.diff(off).min() == 320
    ctx.moves_free(h)


def test_repeated_calls_leave_available_moves_alone(ctx):
    FAST = ctypes.CDLL(fast_lib_path())
    FAST.oracle_fast_moves_available.argtypes = [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 7
    rng = np.random.default_rng(9)
    P, NN = 5000, 24
    slot_off, beg, end = random_rows(rng, P, NN, hot=3)
    h, total = ctx.moves_create(slot_off, beg, end, True, NN)
    first = ctx.moves_schedule(h, 2)
    second = ctx.moves_schedule(h, 2)
    assert np.array_equal(first[0], second[0]) and np.array_equal(first[1], second[1])
    off, node, _, kind = ctx.moves_fetch(h, total)
    nxt = rng.integers(0, 4, P).astype(np.int32)
    node_off, node_parts, best = ctx.moves_available(h, nxt)
    r_off = np.zeros(NN + 1, np.int32); r_parts = np.zeros(P, np.int32); r_best = np.zeros(NN, np.int32)
    assert FAST.oracle_fast_moves_available(P, NN, off.ctypes.data, node.ctypes.data, kind.ctypes.data, nxt.ctypes.data,
                                            r_off.ctypes.data, r_parts.ctypes.data, r_best.ctypes.data) == 0
    assert np.array_equal(node_off, r_off) and np.array_equal(node_parts, r_parts[:r_off[-1]]) and np.array_equal(best, r_best)
    ctx.moves_free(h)


def test_multi_device_context():
    import torch
    G = max(1, min(8, torch.cuda.device_count()))
    mctx = tables.Context(device_ids=list(range(G)))
    rng = np.random.default_rng(13)
    slot_off, beg, end = random_rows(rng, 4000, 16, hot=2)
    h, total = mctx.moves_create(slot_off, beg, end, False, 16)
    for c in (1, 3):
        schedule_both(mctx, h, total, c)
    mctx.moves_free(h)
    mctx.close()
