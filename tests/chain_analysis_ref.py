"""The CPU reference of blance_plan_chains_exposure (include/blance_b200.h), built from oracles already in the tree:
every stage's next rows from the chain reference (chain_util.chain_reference, node ids mapped back to the chain's),
each stage's begMap moves (oracle/fast.c CalcPartitionMoves), their lock-step schedule (tests/schedule_oracle.c) with
its summaries, the vectorised exposure oracle, and a numpy fold of the stages into the span."""
import numpy as np

import chain_util as C
import exposure_oracle as EO
import schedule_oracle as SO
import scenario_exposure_ref as REF
from test_exposure_oracle import calc_moves
from test_scenario_schedule import schedule_summaries

SCHED_PART_FILL = 0                       # part_done_round of a partition outside begMap: no ops


def rebalance(t, next_rows, favor, count, node_has_mover=None, domain_parent=None, oracle=EO.vectorised):
    """(schedule summaries, exposure dict) of the rebalance of tables t (its begMap, constraints and top state) from
    t's prev rows to next_rows at `count`, every per-partition array scattered to [n_parts]."""
    member, beg, end = REF.begmap_rows(t, next_rows)
    slot_off = np.asarray(t.state_slot_off, np.int32)
    off, node, state, kind = calc_moves(slot_off, beg, end, favor)
    NU = t.n_node_ids
    mover = (np.arange(NU) < t.n_nodes).astype(np.uint8) if node_has_mover is None else np.asarray(node_has_mover, np.uint8)
    ro, so, _ = SO.schedule(off, node, kind, NU, max(1, int(count)), mover)
    s = schedule_summaries(off, node, NU, ro, so)
    full = np.full(t.n_parts, SCHED_PART_FILL, np.int32)
    full[member] = s["part_done_round"]
    s["part_done_round"] = full
    e = oracle(slot_off, beg, off, node, state, kind, ro, so, np.asarray(t.state_constraints, np.int32), int(t.top_state), NU, domain_parent)
    for k, fill, dt in REF.PART_FILL:
        f = np.full(t.n_parts, fill, dt)
        f[member] = e[k]
        e[k] = f
    return s, e


def chain_analysis(base, chain, opts, favor, counts, node_has_mover=None, domain_parent=None, oracle=EO.vectorised):
    """One chain's (stages, net, spans): stages[t][k] and net[k] are (schedule summaries, exposure) pairs, spans[k]
    the fold of the stages at counts[k]."""
    ref, _ = C.chain_reference(base, chain, opts, favor)
    cur, stages = base, []
    for t, stage in enumerate(chain):
        x = C.substituted(cur, stage, opts, t)
        stages.append([rebalance(x, ref[t]["next_rows"], favor, c, node_has_mover, domain_parent, oracle) for c in counts])
        cur = C.advance(cur, ref[t]["next_rows"], ref[t]["next_shape"])
    x = C.substituted(base, chain[-1], opts, 0)
    net = [rebalance(x, ref[-1]["next_rows"], favor, c, node_has_mover, domain_parent, oracle) for c in counts]
    spans = [fold([st[k][0] for st in stages], [st[k][1] for st in stages]) for k in range(len(counts))]
    return stages, net, spans


def fold(scheds, expos):
    """The span of blance_chain_span_out from one count's per-stage schedule summaries and exposures (expos may hold
    None: no exposure fields)."""
    G = np.cumsum([0] + [s["rounds"] for s in scheds])[:-1]
    sp = dict(rounds=int(sum(s["rounds"] for s in scheds)), moves_done=int(sum(s["moves_done"] for s in scheds)),
              stuck_parts=int(sum(s["stuck_parts"] for s in scheds)), max_batch=int(max(s["max_batch"] for s in scheds)))
    sp["node_rounds"] = np.sum([s["node_rounds"] for s in scheds], axis=0).astype(np.int32)
    nl = np.zeros_like(scheds[0]["node_last_round"], np.int64)
    pd = np.zeros_like(scheds[0]["part_done_round"], np.int64)
    stuck = np.zeros(pd.shape, bool)
    for g, s in zip(G, scheds):
        l = np.asarray(s["node_last_round"], np.int64)
        nl = np.where(l > 0, g + l, nl)
        d = np.asarray(s["part_done_round"], np.int64)
        stuck |= d < 0
        pd = np.where(d > 0, g + d, pd)
    sp["node_last_round"] = nl
    sp["part_done_round"] = np.where(stuck, -1, pd)
    if expos[0] is None:
        return sp
    peaks = np.array([e["peak"] for e in expos], np.int64)              # [T][6]
    first = np.argmax(peaks == peaks.max(axis=0), axis=0)
    sp["peak"] = peaks.max(axis=0)
    sp["peak_stage"] = first.astype(np.int32)
    sp["peak_round"] = np.array([expos[t]["peak_round"][m] for m, t in enumerate(first)], np.int32)
    sp["area"] = np.sum([e["area"] for e in expos], axis=0).astype(np.int64)
    mins = np.array([e["part_min_copies"] for e in expos], np.int64)
    big = np.where(mins < 0, np.iinfo(np.int64).max, mins).min(axis=0)
    sp["part_min_copies"] = np.where(big == np.iinfo(np.int64).max, -1, big).astype(np.int32)
    sp["part_no_top"] = np.sum([e["part_no_top"] for e in expos], axis=0).astype(np.int32)
    sp["part_flags"] = np.bitwise_or.reduce([e["part_flags"] for e in expos], axis=0).astype(np.uint8)
    if "dom_peak" in expos[0]:
        dp = np.array([e["dom_peak"] for e in expos], np.int64)
        first = np.argmax(dp == dp.max(axis=0), axis=0)
        sp["dom_peak"] = dp.max(axis=0)
        sp["dom_peak_stage"] = first.astype(np.int32)
        sp["dom_peak_round"] = np.array([expos[t]["dom_peak_round"][v] for v, t in enumerate(first)], np.int32)
    return sp


def assert_span(got, want, what=""):
    for k, w in want.items():
        assert k in got, (what, k)
        assert np.array_equal(np.asarray(got[k]), np.asarray(w)), (what, k, got[k], w)
