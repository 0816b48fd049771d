"""Each node's load while a rebalance runs (blance_moves_load), CPU side: the literal replay against the vectorised
oracle on random move lists scheduled by tests/schedule_oracle.c, hand-derived cases, the reference's
CalcPartitionMoves goldens replayed as one-partition rebalances, the argument errors that need no device, and what
the load kernels compile to."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

import load_oracle as LO
import schedule_oracle as SO
from test_exposure_oracle import ADD, DEL, DEMOTE, NONE, PROMOTE, calc_moves, random_case
from test_sass_guard import kernels  # noqa: F401  (the parsed SASS, a module-scoped fixture)

from blance_b200 import abi, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_WEIGHT = 999999999


def random_weights(rng, P, kind):
    """None (every partition 1), small weights, or weights with 0 and 999999999 mixed in."""
    if kind == 0:
        return None
    w = rng.integers(0, 5, P)
    if kind == 2:
        w[rng.random(P) < 0.2] = 0
        w[rng.random(P) < 0.1] = MAX_WEIGHT
    return w.astype(np.int64)


def both(slot_off, beg, moves, sched, NN, w=None):
    off, node, state, kind = moves
    ro, so = sched
    args = (slot_off, beg, off, node, state, kind, ro, so, NN, w)
    return LO.replay(*args), LO.vectorised(*args)


@pytest.mark.parametrize("chunk", range(4))
def test_replay_equals_the_vectorised_oracle(chunk):
    rng = np.random.default_rng(900 + chunk)
    for trial in range(40):
        slot_off, beg, end, _, _, NN = random_case(rng)
        S = len(slot_off) - 1
        n_visit = int(rng.integers(1, S + 1)) if trial % 3 == 0 else S
        moves = calc_moves(slot_off, beg, end, trial % 2 == 0, n_visit)
        mover = (rng.random(NN) >= 0.15).astype(np.uint8) if trial % 4 == 1 else None
        NU = NN - 2 if trial % 5 == 2 else NN                   # ids NU .. NN - 1 lie outside the node range
        w = random_weights(rng, beg.shape[0], trial % 3)
        for c in (1, 2, 4):
            ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], NU, c, None if mover is None else mover[:NU])
            lit, vec = both(slot_off, beg, moves, (ro, so), NU, w)
            LO.assert_equal(vec, lit, (chunk, trial, c))
            assert (lit["node_peak"] >= np.maximum(lit["node_beg"], lit["node_end"])).all()


def one_partition(slot_off, beg_row, ops, NN, w=None):
    """A rebalance of one partition whose ops are `ops` [(node, state, kind)], one op per round."""
    off = np.array([0, len(ops)], np.int64)
    node = np.array([o[0] for o in ops], np.int32)
    state = np.array([o[1] for o in ops], np.uint8)
    kind = np.array([o[2] for o in ops], np.uint8)
    ro, so, _ = SO.schedule(off, node, kind, NN, 1)
    return both(np.asarray(slot_off, np.int32), np.asarray([beg_row], np.int32), (off, node, state, kind), (ro, so), NN,
                None if w is None else [w])


def test_primary_moves_overshoot_without_favor_min_nodes():
    # partition 0's primary moves a -> b and partition 1's b -> a.  Without favorMinNodes each add runs first (round
    # 0) and each del after it (round 1), so at t = 1 both nodes hold both primaries: w more than at either end.  With
    # favorMinNodes the dels run first and nothing overshoots.
    slot_off, a, b, w = [0, 1, 2], 0, 1, 7
    beg, end = np.array([[a, -1], [b, -1]], np.int32), np.array([[b, -1], [a, -1]], np.int32)
    for favor in (False, True):
        moves = calc_moves(slot_off, beg, end, favor)
        ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], 2, 1)
        lit, vec = both(np.asarray(slot_off, np.int32), beg, moves, (ro, so), 2, [w, w])
        LO.assert_equal(vec, lit)
        assert lit["rounds"] == 2
        assert lit["node_beg"][2].tolist() == [w, w] and lit["node_end"][2].tolist() == [w, w]
        if favor:
            assert lit["over_max"] == 0 and lit["over_node"] == a
            assert lit["node_peak"][2].tolist() == [w, w] and lit["node_peak_round"][2].tolist() == [0, 0]
        else:
            assert lit["over_max"] == w and lit["over_node"] == a
            assert lit["node_peak"][2].tolist() == [2 * w, 2 * w] and lit["node_peak_round"][2].tolist() == [1, 1]
            assert lit["node_peak"][0].tolist() == [2 * w, 2 * w]


def test_one_primary_move_never_overshoots_a_node():
    # a single move a -> b: a's largest load is its start load and b's its end load, with or without favorMinNodes
    slot_off, a, b, w = [0, 1, 2], 0, 1, 7
    for favor, peak_round in ((False, [0, 1]), (True, [0, 2])):
        moves = calc_moves(slot_off, [[a, -1]], [[b, -1]], favor)
        ro, so, _ = SO.schedule(moves[0], moves[1], moves[3], 2, 1)
        lit, vec = both(np.asarray(slot_off, np.int32), np.asarray([[a, -1]], np.int32), moves, (ro, so), 2, [w])
        LO.assert_equal(vec, lit)
        assert lit["over_max"] == 0 and lit["node_peak_round"][2].tolist() == peak_round


def test_replica_swap():
    # primary a, replica b -> primary b, replica a: promote b, demote a; every node holds one copy throughout
    lit, vec = one_partition([0, 1, 2], [0, 1], [(1, 0, PROMOTE), (0, 1, DEMOTE)], 2, 3)
    LO.assert_equal(vec, lit)
    assert lit["node_beg"].tolist() == [[3, 0], [0, 3], [3, 3]]
    assert lit["node_end"].tolist() == [[0, 3], [3, 0], [3, 3]]
    assert lit["over_max"] == 0 and lit["node_peak"][2].tolist() == [3, 3]
    assert lit["node_peak"][0].tolist() == [3, 3] and lit["node_peak_round"][0].tolist() == [0, 1]


def test_stuck_partition_end_is_not_the_end_map():
    # primary a -> b with b without a mover (favorMinNodes): a is deleted, b's add never runs
    moves = calc_moves([0, 1], [[0]], [[1]], True)
    ro, so, sc = SO.schedule(moves[0], moves[1], moves[3], 2, 1, np.array([1, 0], np.uint8))
    assert sc["stuck_parts"] == 1 and sc["rounds"] == 1
    lit, vec = both(np.array([0, 1], np.int32), np.array([[0]], np.int32), moves, (ro, so), 2)
    LO.assert_equal(vec, lit)
    assert lit["node_end"][1].tolist() == [0, 0]               # the end map would put 1 on b
    assert lit["node_beg"][1].tolist() == [1, 0] and lit["over_max"] == 0


def test_node_listed_twice_and_ids_outside_the_range():
    # node 0 twice as a replica counts twice until its op; node 5 outside [0, 3) counts nowhere
    lit, vec = one_partition([0, 1, 3], [5, 0, 0], [(1, 0, ADD), (0, NONE, DEL)], 3, 2)
    LO.assert_equal(vec, lit)
    assert lit["node_beg"].tolist() == [[0, 0, 0], [4, 0, 0], [4, 0, 0]]
    assert lit["node_end"].tolist() == [[0, 2, 0], [0, 0, 0], [0, 2, 0]]
    assert lit["node_peak"][2].tolist() == [4, 2, 0] and lit["node_peak_round"][2].tolist() == [0, 1, 0]
    assert lit["over_max"] == 0 and lit["over_node"] == 0


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
        NN = max(1, len(nodes))
        lit, vec = one_partition(slot_off, row, ops, NN, 5)
        LO.assert_equal(vec, lit, c["index"])
        # direct count over the prefix maps of the expected ops: each node's copies at every t
        m = {n: [s for s in states for x in c["before"].get(s, []) if x == n] for n in nodes}
        per_t = [{n: len(v) for n, v in m.items()}]
        for e in c["exp"]:
            m[e["node"]] = [] if e["state"] == "" else [e["state"]]
            per_t.append({n: len(v) for n, v in m.items()})
        S = len(states)
        for n in nodes:
            series = [5 * x[n] for x in per_t]
            assert lit["node_peak"][S][ids[n]] == max(series), c["index"]
            assert lit["node_peak_round"][S][ids[n]] == series.index(max(series)), c["index"]
            assert lit["node_end"][S][ids[n]] == series[-1], c["index"]


def test_abi_errors_without_a_device():
    lib = abi.capi()
    l_in, out = abi.LoadIn(None, None), abi.LoadOut()
    for args in ((None, None, ctypes.byref(l_in), ctypes.byref(out)), (None, None, None, None),
                 (None, None, None, ctypes.byref(out)), (None, None, ctypes.byref(l_in), None)):
        assert lib.blance_moves_load(*args) == -1
        assert lib.blance_last_error(None) == b"blance_moves_load: ctx, moves, in or out is NULL"
    assert ctypes.sizeof(abi.LoadIn) == 16 and ctypes.sizeof(abi.LoadOut) == 56       # the layout of the header


def test_struct_layout_matches_header(tmp_path):
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    int main(void) { printf("%zu %zu %zu %zu %zu %zu\n", sizeof(blance_load_in), sizeof(blance_load_out),
                            offsetof(blance_load_out, node_peak_round), offsetof(blance_load_out, over_max),
                            offsetof(blance_load_out, over_node), offsetof(blance_load_out, kernel_ms)); return 0; }
    '''
    c = tmp_path / "p.c"
    c.write_text(probe)
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")], check=True)
    got = list(map(int, subprocess.run([str(tmp_path / "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    assert got == [ctypes.sizeof(abi.LoadIn), ctypes.sizeof(abi.LoadOut), abi.LoadOut.node_peak_round.offset,
                   abi.LoadOut.over_max.offset, abi.LoadOut.over_node.offset, abi.LoadOut.kernel_ms.offset]


def test_the_library_needs_no_second_native_library():
    out = subprocess.run(["readelf", "-d", build.lib_path()], stdout=subprocess.PIPE, text=True, check=True).stdout
    assert "NEEDED" in out and "libblance_b200_load.so" not in out


def test_load_kernels_in_the_library_use_reductions_and_no_atomics(kernels):  # noqa: F811
    own = {k: "\n".join(b) for k, b in kernels.items() if "k_load_" in k}
    assert len(own) == 5, sorted(own)          # walk<0|1>, init, peak, final
    for k, body in own.items():
        assert "ATOMG" not in body, k
    for name in ("k_load_walkILi0E", "k_load_peak", "k_load_final"):
        assert any("REDG" in b for k, b in own.items() if name in k), name
    walk0 = [b for k, b in own.items() if "k_load_walkILi0E" in k][0]
    assert "MATCH" in walk0 and "REDUX" in walk0   # lanes of one index merged before their RED
