"""The exposure of a rebalance (blance_moves_exposure), CPU side: the literal replay against the vectorised oracle on
random move lists scheduled by tests/schedule_oracle.c, hand-derived cases, the reference's CalcPartitionMoves
goldens replayed as one-partition rebalances, and the argument errors that need no device."""
import ctypes
import json
import os

import numpy as np
import pytest

import exposure_oracle as EO
import schedule_oracle as SO
from test_fast_oracle import FAST

from blance_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST.oracle_fast_calc_partition_moves.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 4


def calc_moves(slot_off, beg, end, favor, n_visit=None):
    """CSR CalcPartitionMoves of every row pair (oracle/fast.c): op_off, op_node, op_state, op_kind."""
    slot_off = np.ascontiguousarray(slot_off, np.int32)
    beg = np.ascontiguousarray(beg, np.int32)
    end = np.ascontiguousarray(end, np.int32)
    P, S = beg.shape[0], len(slot_off) - 1
    MO = max(1, 2 * int(slot_off[-1]))
    on = np.zeros((P, MO), np.int32); os_ = np.zeros((P, MO), np.uint8); ok = np.zeros((P, MO), np.uint8)
    cnt = np.zeros(max(P, 1), np.int32)
    if P:
        assert FAST.oracle_fast_calc_partition_moves(P, S, S if n_visit is None else n_visit, slot_off.ctypes.data, beg.ctypes.data,
                                                     end.ctypes.data, int(favor), MO, on.ctypes.data, os_.ctypes.data,
                                                     ok.ctypes.data, cnt.ctypes.data) == 0
    cnt = cnt[:P]
    mask = np.arange(MO)[None, :] < cnt[:, None]
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    return off, on[mask], os_[mask], ok[mask]


def random_forest(rng, NN, depth):
    """parent [NN + n_domains]: nodes hang under a random chain of up to `depth` inner levels."""
    inner = []
    parent = []
    level = [-1]
    for _ in range(depth):
        nxt = []
        for _ in range(int(rng.integers(1, 4))):
            inner.append(int(rng.choice(level)))
            nxt.append(NN + len(inner) - 1)
        level = nxt
    for _ in range(NN):
        parent.append(int(rng.choice(level)) if rng.random() < 0.9 else -1)
    return np.asarray(parent + inner, np.int32)


def random_case(rng, P=None, NN=None):
    S = int(rng.integers(1, 4))
    caps = rng.integers(1, 4, S)
    slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
    SL = int(slot_off[-1])
    P = int(rng.integers(0, 40)) if P is None else P
    NN = int(rng.integers(2, 9)) if NN is None else NN

    def rows(dup):
        r = np.full((P, SL), -1, np.int32)
        for p in range(P):
            perm = rng.permutation(max(NN, SL))[:SL] % NN
            for s in range(S):
                n = int(rng.integers(0, caps[s] + 1))
                r[p, slot_off[s]:slot_off[s] + n] = perm[slot_off[s]:slot_off[s] + n]
            if dup and SL > 1 and rng.random() < 0.2:          # a node listed twice
                i, j = rng.choice(SL, 2, replace=False)
                if r[p, i] >= 0 and r[p, j] >= 0:
                    r[p, j] = r[p, i]
        return r
    beg, end = rows(True), rows(False)
    same = rng.random(P) < 0.15                                  # partitions without ops
    end[same] = beg[same]
    cons = rng.integers(0, 3, S).astype(np.int32)
    top = int(rng.integers(-1, S))
    return slot_off, beg, end, cons, top, NN


def both(slot_off, beg, moves, sched, cons, top, NN, parent=None):
    off, node, state, kind = moves
    ro, so = sched
    args = (slot_off, beg, off, node, state, kind, ro, so, cons, top, NN, parent)
    return EO.replay(*args), EO.vectorised(*args)


@pytest.mark.parametrize("chunk", range(4))
def test_replay_equals_the_vectorised_oracle(chunk):
    rng = np.random.default_rng(700 + chunk)
    for trial in range(40):
        slot_off, beg, end, cons, top, NN = random_case(rng)
        S = len(slot_off) - 1
        n_visit = int(rng.integers(1, S + 1)) if trial % 3 == 0 else S
        moves = calc_moves(slot_off, beg, end, trial % 2 == 0, n_visit)
        mover = (rng.random(NN) >= 0.15).astype(np.uint8) if trial % 4 == 1 else None
        parent = random_forest(rng, NN, int(rng.integers(0, 17))) if trial % 2 else None
        for c in (1, 2, 4):
            ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], NN, c, mover)
            lit, vec = both(slot_off, beg, moves, (ro, so), cons, top, NN, parent)
            EO.assert_equal(vec, lit, (chunk, trial, c))


def one_partition(slot_off, beg_row, ops, cons, top, NN):
    """A rebalance of one partition whose ops are `ops` [(node, state, kind)], one op per round."""
    off = np.array([0, len(ops)], np.int64)
    node = np.array([o[0] for o in ops], np.int32)
    state = np.array([o[1] for o in ops], np.uint8)
    kind = np.array([o[2] for o in ops], np.uint8)
    ro, so, _ = SO.schedule(off, node, kind, NN, 1)
    return both(np.asarray(slot_off, np.int32), np.asarray([beg_row], np.int32), (off, node, state, kind), (ro, so), cons, top, NN)


ADD, DEL, PROMOTE, DEMOTE, NONE = 0, 1, 2, 3, 0xFF


def test_primary_move_favor_min_nodes():
    # primary a -> b: favorMinNodes gives a del, b add (no copy in between); otherwise b add, a del (two primaries)
    slot_off, a, b = [0, 1, 2], 0, 1
    for favor, want in ((True, "NO_COPY"), (False, "MULTI_TOP")):
        moves = calc_moves(slot_off, [[a, -1]], [[b, -1]], favor)
        ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], 2, 1)
        lit, vec = both(np.asarray(slot_off, np.int32), np.asarray([[a, -1]], np.int32), moves, (ro, so), [1, 0], 0, 2)
        EO.assert_equal(vec, lit)
        m = EO.METRICS.index(want)
        assert lit["rounds"] == 2 and lit["series"][m].tolist() == [0, 1, 0], favor
        assert lit["peak"][m] == 1 and lit["peak_round"][m] == 1
        other = EO.METRICS.index("MULTI_TOP" if favor else "NO_COPY")
        assert lit["series"][other].tolist() == [0, 0, 0]
        assert lit["part_min_copies"].tolist() == [0 if favor else 1]
        assert lit["dom_peak"].tolist() == [1, 1]             # each node alone holds the partition at some t


def test_replica_swap():
    # primary a, replica b -> primary a, replica c: add c, then del b; three copies in between, never fewer than two
    lit, vec = one_partition([0, 1, 2], [0, 1], [(2, 1, ADD), (1, NONE, DEL)], [1, 1], 0, 3)
    EO.assert_equal(vec, lit)
    assert lit["series"][EO.METRICS.index("COPIES")].tolist() == [2, 3, 2]
    assert lit["peak"][EO.METRICS.index("ONE_COPY")] == 0 and lit["part_min_copies"].tolist() == [2]
    assert lit["dom_peak"].tolist() == [0, 0, 0]


def test_stuck_partition_keeps_its_state():
    # primary a -> b with b without a mover (favorMinNodes): a is deleted, b's add never runs
    moves = calc_moves([0, 1], [[0]], [[1]], True)
    ro, so, sc = SO.schedule(moves[0], moves[1], moves[3], 2, 1, np.array([1, 0], np.uint8))
    assert sc["stuck_parts"] == 1 and sc["rounds"] == 1
    lit, vec = both(np.array([0, 1], np.int32), np.array([[0]], np.int32), moves, (ro, so), [1], 0, 2)
    EO.assert_equal(vec, lit)
    assert lit["series"][EO.METRICS.index("NO_COPY")].tolist() == [0, 1]
    assert lit["part_no_top"].tolist() == [1] and lit["part_flags"].tolist() == [1 | 4 | 8 | 16 | 32]


def test_golden_moves_as_one_partition_rebalances():
    with open(os.path.join(ROOT, "tests", "golden", "moves_cases.json")) as f:
        cases = json.load(f)["calcPartitionMoves"]
    kinds = {"add": ADD, "del": DEL, "promote": PROMOTE, "demote": DEMOTE}
    for c in cases:
        states = c["states"]
        caps = [max(1, len(c["before"].get(s, []))) for s in states]
        slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
        nodes = sorted({n for lst in list(c["before"].values()) + list(c["after"].values()) for n in lst})
        ids = {n: i for i, n in enumerate(nodes)}
        row = np.full(int(slot_off[-1]), -1, np.int32)
        for s, name in enumerate(states):
            for j, n in enumerate(c["before"].get(name, [])):
                row[slot_off[s] + j] = ids[n]
        ops = [(ids[e["node"]], NONE if e["state"] == "" else states.index(e["state"]), kinds[e["op"][0]]) for e in c["exp"]]
        lit, vec = one_partition(slot_off, row, ops, [0] * len(states), -1, max(1, len(nodes)))
        EO.assert_equal(vec, lit, c["index"])
        # direct count over the prefix maps of the expected ops
        m = {n: [s for s in states for x in c["before"].get(s, []) if x == n] for n in nodes}
        counts = [sum(len(v) for v in m.values())]
        for e in c["exp"]:
            m[e["node"]] = [] if e["state"] == "" else [e["state"]]
            counts.append(sum(len(v) for v in m.values()))
        assert lit["part_min_copies"].tolist() == [min(counts)], c["index"]
        assert lit["series"][EO.METRICS.index("COPIES")].tolist() == counts, c["index"]


def test_abi_errors_without_a_device():
    lib = abi.capi()
    e_in = abi.ExposureIn(None, -1, 0, None)
    out = abi.ExposureOut()
    assert lib.blance_moves_exposure(None, None, ctypes.byref(e_in), ctypes.byref(out)) == -1
    assert b"NULL" in lib.blance_last_error(None)
    assert ctypes.sizeof(abi.ExposureOut) == 184 and ctypes.sizeof(abi.ExposureIn) == 24   # the layout of the header
