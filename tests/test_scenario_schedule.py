"""The schedule summaries of blance_plan_scenarios_schedule (include/blance_b200.h), CPU side: one helper derives
node_rounds, node_last_round, part_done_round, stuck_parts and max_batch from a schedule's round_off / sched_op and
its CSR move lists, and it must equal a direct reading of schedule_oracle.go_reading's batches; the C struct layout
matches the ctypes one; the new entry point rejects bad arguments without a device."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import schedule_oracle as SO
from test_schedule_oracle import COUNTS, random_lists

from blance_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def schedule_summaries(off, node, n_node_ids, round_off, sched_op):
    """The blance_scenario_schedule_out summaries a schedule implies: node_rounds[q] = rounds with an op on q,
    node_last_round[q] = 1 + the last such round (0 = none), part_done_round[p] = 1 + the round of p's last op when
    all its ops ran, 0 without ops, -1 when ops are left (stuck); stuck_parts; max_batch = most ops of one node in one
    round."""
    off = np.asarray(off, np.int64)
    so = np.asarray(sched_op, np.int64)
    ro = np.asarray(round_off, np.int64)
    P = len(off) - 1
    node_rounds = np.zeros(n_node_ids, np.int32)
    node_last = np.zeros(n_node_ids, np.int32)
    max_batch = 0
    for r in range(len(ro) - 1):
        nodes = np.asarray(node, np.int64)[so[ro[r]:ro[r + 1]]]
        if not len(nodes):
            continue
        q, c = np.unique(nodes, return_counts=True)
        node_rounds[q] += 1
        node_last[q] = r + 1
        max_batch = max(max_batch, int(c.max()))
    n_ops = np.diff(off)
    part = np.searchsorted(off, so, side="right") - 1
    rnd = np.searchsorted(ro, np.arange(len(so)), side="right") - 1
    done = np.bincount(part, minlength=P) if len(so) else np.zeros(P, np.int64)
    last = np.zeros(P, np.int64)
    if len(so):
        np.maximum.at(last, part, rnd + 1)
    part_done = np.where(n_ops == 0, 0, np.where(done == n_ops, last, -1)).astype(np.int32)
    return dict(rounds=len(ro) - 1, moves_done=len(so), stuck_parts=int((part_done < 0).sum()), max_batch=max_batch,
                node_rounds=node_rounds, node_last_round=node_last, part_done_round=part_done)


def go_summaries(off, node, n_node_ids, rounds):
    """The same summaries read straight from go_reading's batches [[(node, [op, ...]), ...], ...]."""
    P = len(off) - 1
    node_rounds = np.zeros(n_node_ids, np.int32)
    node_last = np.zeros(n_node_ids, np.int32)
    left = np.diff(np.asarray(off, np.int64)).astype(np.int64)
    part_done = np.zeros(P, np.int32)
    max_batch, moves = 0, 0
    for r, batches in enumerate(rounds):
        for q, ops in batches:
            node_rounds[q] += 1
            node_last[q] = r + 1
            max_batch = max(max_batch, len(ops))
            moves += len(ops)
            for o in ops:
                p = int(np.searchsorted(off, o, side="right") - 1)
                left[p] -= 1
                if left[p] == 0:
                    part_done[p] = r + 1
    part_done[left > 0] = -1
    return dict(rounds=len(rounds), moves_done=moves, stuck_parts=int((left > 0).sum()), max_batch=max_batch,
                node_rounds=node_rounds, node_last_round=node_last, part_done_round=part_done)


def assert_same_summaries(a, b, what=None):
    for k in ("rounds", "moves_done", "stuck_parts", "max_batch"):
        assert a[k] == b[k], (what, k, a[k], b[k])
    for k in ("node_rounds", "node_last_round", "part_done_round"):
        assert np.array_equal(a[k], b[k]), (what, k)


@pytest.mark.parametrize("chunk", range(3))
def test_summary_helper_equals_the_go_reading(chunk):
    rng = np.random.default_rng(700 + chunk)
    for trial in range(60):
        off, node, kind, NN, mover = random_lists(rng, long_node=trial % 2 == 0)
        for c in COUNTS:
            ro, so, sc = SO.schedule(off, node, kind, NN, c, mover)
            got = schedule_summaries(off, node, NN, ro, so)
            assert_same_summaries(got, go_summaries(off, node, NN, SO.go_reading(off, node, kind, NN, c, mover)), (chunk, trial, c))
            assert {k: got[k] for k in sc} == sc


def test_summaries_of_a_node_without_a_mover():
    """p0: add on 0 then del on 1 (no mover): stuck after one round; p1: no ops; p2: promote on 0."""
    off = np.array([0, 2, 2, 3], np.int64)
    node = np.array([0, 1, 0], np.int32)
    kind = np.array([0, 1, 2], np.uint8)
    mover = np.array([1, 0], np.uint8)
    ro, so, sc = SO.schedule(off, node, kind, 2, 1, mover)
    s = schedule_summaries(off, node, 2, ro, so)
    assert s["part_done_round"].tolist() == [-1, 0, 1] and s["stuck_parts"] == 1
    assert s["node_rounds"].tolist() == [2, 0] and s["node_last_round"].tolist() == [2, 0] and s["rounds"] == 2


def test_scenario_schedule_struct_layout_matches_header():
    probe = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "blance_b200.h"
    #define F(f) offsetof(blance_scenario_schedule_out, f)
    int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(blance_scenario_schedule_out), F(rounds), F(moves_done),
                            F(stuck_parts), F(max_batch), F(node_rounds), F(node_last_round), F(part_done_round)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")], check=True)
        out = list(map(int, subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()))
    S = api.ScenarioScheduleOut
    assert out == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in ("rounds", "moves_done", "stuck_parts", "max_batch",
                                                                       "node_rounds", "node_last_round", "part_done_round")]


def test_bad_schedule_arguments_without_a_device():
    lib = api.capi()
    base = api.PlanIn()
    scs = (api.Scenario * 1)()
    outs = (api.ScenarioOut * 1)()
    sch = (api.ScenarioScheduleOut * 1)()
    counts = (ctypes.c_int32 * 1)(1)
    assert lib.blance_plan_scenarios_schedule(None, ctypes.byref(base), 1, scs, None, 0, 0, 1, counts, None, outs, sch) == -1
    assert b"NULL" in lib.blance_last_error(None)
