"""The lock-step schedule of blance_moves_schedule (include/blance_b200.h), CPU side: the serial oracle
(tests/schedule_oracle.c) against a direct Python reading of orchestrate.go:482-504, 509-591, 749-763 and 177-186,
the reference's TestOrchestrateConcurrentMoves batches through the oracle, the schedule's invariants, and the C ABI
surface that needs no device (struct layout, NULL arguments, SASS of the new kernels)."""
import ctypes
import json
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import schedule_oracle as SO
from oracle_loader import literal

from blance_b200 import api, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "orchestrate_concurrency_cases.json")
KINDS = ["add", "del", "promote", "demote"]
COUNTS = (-1, 0, 1, 2, 3, 7, 64)


def random_lists(rng, long_node=True):
    """CSR move lists with common weight ties (mostly adds), partitions without ops, a few node ids without a
    mover, and (long_node) one node whose list is much longer than most counts."""
    P, NN = int(rng.integers(0, 60)), int(rng.integers(1, 9))
    lens = rng.integers(0, 5, P)
    lens[rng.random(P) < 0.15] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    T = int(off[-1])
    node = rng.integers(0, NN, T).astype(np.int32)
    if long_node and T:
        node[rng.random(T) < 0.5] = 0
    kind = rng.choice(4, T, p=[0.6, 0.2, 0.15, 0.05]).astype(np.uint8)
    mover = (rng.random(NN) >= 0.15).astype(np.uint8)
    mover[0] = 1
    return off, node, kind, NN, mover


def check_invariants(off, node, kind, NN, c, mover, ro, so, sc):
    T = int(off[-1])
    assert len(so) == sc["moves_done"] == ro[-1] and len(ro) == sc["rounds"] + 1
    assert len(set(so.tolist())) == len(so)                              # each op at most once
    part = np.searchsorted(off, so, side="right") - 1
    rnd = np.searchsorted(ro, np.arange(len(so)), side="right") - 1
    last = {}
    for i, (o, p, r) in enumerate(zip(so.tolist(), part.tolist(), rnd.tolist())):
        prev = last.get(p)
        assert o == (off[p] if prev is None else prev[0] + 1)              # a partition's ops in list order
        assert prev is None or r > prev[1]                                 # ... in strictly increasing rounds
        last[p] = (o, r)
    cap = max(1, c)
    for r in range(sc["rounds"]):
        nodes = node[so[ro[r]:ro[r + 1]]]
        assert (np.diff(nodes) >= 0).all()                                 # batches in ascending node id
        assert np.bincount(nodes, minlength=NN).max() <= cap               # at most max(1, c) per node and round
        assert mover[nodes].all()
    # moves_done + the ops stuck partitions still have from their cursor on == total_ops
    done = np.bincount(part, minlength=len(off) - 1) if len(so) else np.zeros(len(off) - 1, np.int64)
    left = (np.diff(off) - done)
    stuck = left > 0
    assert int(stuck.sum()) == sc["stuck_parts"]
    assert sc["moves_done"] + int(left[stuck].sum()) == T
    for p in np.nonzero(stuck)[0]:
        assert not mover[node[off[p] + done[p]]]


@pytest.mark.parametrize("chunk", range(4))
def test_oracle_equals_the_go_statements_on_random_lists(chunk):
    rng = np.random.default_rng(100 + chunk)
    for trial in range(80):
        off, node, kind, NN, mover = random_lists(rng, long_node=trial % 2 == 0)
        for c in COUNTS:
            ro, so, sc = SO.schedule(off, node, kind, NN, c, mover)
            want_ro, want_so = SO.flatten(SO.go_reading(off, node, kind, NN, c, mover))
            assert np.array_equal(ro, want_ro) and np.array_equal(so, want_so), (chunk, trial, c)
            check_invariants(off, node, kind, NN, c, mover, ro, so, sc)


def test_swap_remove_decides_ties():
    """Adds on p1, p2, p3 at c = 2: p1 is picked, p3 takes its place and is picked next - not p2."""
    off = np.array([0, 1, 2, 3], np.int64)
    ro, so, sc = SO.schedule(off, np.zeros(3, np.int32), np.zeros(3, np.uint8), 1, 2)
    assert so.tolist() == [0, 2, 1] and ro.tolist() == [0, 2, 3] and sc["max_batch"] == 2


def test_every_node_without_a_mover():
    rng = np.random.default_rng(5)
    off, node, kind, NN, _ = random_lists(rng)
    ro, so, sc = SO.schedule(off, node, kind, NN, 2, np.zeros(NN, np.uint8))
    assert sc["rounds"] == 0 and len(so) == 0 and ro.tolist() == [0]
    assert sc["stuck_parts"] == int((np.diff(off) > 0).sum())


# ---- TestOrchestrateConcurrentMoves (orchestrate_test.go:452-1047) --------------------------------------------

def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)


def golden_lists(c):
    """The CSR move lists OrchestrateMoves seeds (orchestrate.go:263-287), through the literal CalcPartitionMoves:
    partitions = begMap's keys in byte order, node ids = nodesAll first, states in sortStateNames order."""
    model = c["model"]
    states = sorted(model, key=lambda k: (model[k]["priority"], k))
    names = sorted(c["begMap"])
    nodes = list(dict.fromkeys(c["nodesAll"]))
    n_movers = len(nodes)
    off, node, state, kind = [0], [], [], []
    for p in names:
        end = (c["endMap"].get(p) or {"nodesByState": {}})["nodesByState"]
        for n, s, op in literal().calc_partition_moves(states, c["begMap"][p]["nodesByState"], end, False):
            if n not in nodes:
                nodes.append(n)
            node.append(nodes.index(n)); state.append(s); kind.append(KINDS.index(op))
        off.append(len(node))
    mover = np.array([i < n_movers for i in range(len(nodes))], np.uint8)
    return names, nodes, np.array(off, np.int64), np.array(node, np.int32), state, np.array(kind, np.uint8), mover


def golden_batch(c, rounds):
    """The (skipCallbacks + 1)-th AssignPartitionsFunc call on expNode: (partitions, states, ops) or None."""
    seen = 0
    for batches in rounds:
        for node, parts, states, ops in batches:
            if node != c["expNode"]:
                continue
            if seen == c["skipCallbacks"]:
                return parts, states, ops
            seen += 1
    return None


def check_golden_batch(c, got):
    assert got is not None, c["label"]
    parts, states, ops = got
    assert len(parts) == c["expConcurrentMovesCount"], c["label"]
    assert sorted(parts) == c["expMovePartitions"], c["label"]
    assert sorted(states) == c["expMoveStates"], c["label"]
    assert list(ops) == c["expMoveOps"], c["label"]


def test_golden_fixture_has_the_six_cases():
    cases = golden_cases()
    assert [c["index"] for c in cases] == [0, 1, 3, 4, 5, 6]


@pytest.mark.parametrize("c", golden_cases(), ids=lambda c: "%d-%s" % (c["index"], c["label"].replace(" ", "_")))
def test_golden_batches_through_the_oracle(c):
    names, nodes, off, node, state, kind, mover = golden_lists(c)
    ro, so, sc = SO.schedule(off, node, kind, len(nodes), c["maxConcurrentMoves"], mover)
    rounds = []
    for r in range(sc["rounds"]):
        batches = []
        for o in so[ro[r]:ro[r + 1]].tolist():
            p = int(np.searchsorted(off, o, side="right") - 1)
            if not batches or batches[-1][0] != nodes[node[o]]:
                batches.append((nodes[node[o]], [], [], []))
            batches[-1][1].append(names[p]); batches[-1][2].append(state[o]); batches[-1][3].append(KINDS[kind[o]])
        rounds.append(batches)
    check_golden_batch(c, golden_batch(c, rounds))


# ---- the C ABI without a device -----------------------------------------------------------------------------

def test_schedule_struct_layout_matches_header():
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    int main(void) { printf("%zu %zu %zu %zu %zu %zu\n", sizeof(blance_schedule_out), offsetof(blance_schedule_out, rounds),
                            offsetof(blance_schedule_out, moves_done), offsetof(blance_schedule_out, stuck_parts),
                            offsetof(blance_schedule_out, max_batch), offsetof(blance_schedule_out, device_ms)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")], check=True)
        out = list(map(int, subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    S = api.ScheduleOut
    assert out == [ctypes.sizeof(S), S.rounds.offset, S.moves_done.offset, S.stuck_parts.offset, S.max_batch.offset,
                   S.device_ms.offset]


def test_null_arguments_are_invalid_without_a_device():
    lib = api.capi()
    out = api.ScheduleOut()
    assert lib.blance_moves_schedule(None, None, 1, None, ctypes.byref(out)) == -1
    assert lib.blance_moves_schedule(None, ctypes.c_void_p(8), 1, None, None) == -1
    assert lib.blance_moves_schedule_fetch(None, None, None, None) == -1
    assert b"NULL" in lib.blance_last_error(None)


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def test_wave_kernels_issue_value_less_atomics_as_red():
    """The schedule engine's kernels (k_wave_*, wave_schedule.cuh) discard their atomics' results: the per-node op
    histogram, the stuck counts and the per-instance summaries must compile to RED, not to ATOM with a return value
    the warp would wait for."""
    try:
        txt = subprocess.run([CUOBJDUMP, "-sass", build.lib_path()], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300).stdout
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump is not available")
    kernels, name = {}, None
    for line in txt.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,6}\*/", line):
            kernels[name].append(line)
    sched = {k: "\n".join(v) for k, v in kernels.items() if "k_wave_" in k}
    if not sched:
        pytest.skip("cuobjdump printed no SASS")
    assert len(sched) == 6, sorted(sched)
    for k, body in sched.items():
        assert not re.search(r"ATOMG?\.\S+ PT, RZ,", body), k
    for want in ("k_wave_pick", "k_wave_first", "k_wave_node_ops"):
        body = next(b for k, b in sched.items() if want in k)
        assert re.search(r"\bREDG?\.", body), want
