"""blance_plan_chains_exposure (include/blance_b200.h), CPU side: the ctypes declaration against the header, every
argument error with a NULL context (no device needed), the Python wrapper's own errors, and the CPU reference of the
per-stage schedules, exposures and spans (tests/chain_analysis_ref.py) against a literal replay of every stage."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import chain_analysis_ref as CA
import exposure_oracle as EO
import schedule_oracle as SO
from test_chains_gpu import random_chains
from test_exposure_oracle import calc_moves, random_forest
from test_scenario_schedule import assert_same_summaries, go_summaries
from test_scenarios_gpu import random_base

import chain_util as C
import scenario_exposure_ref as REF
from blance_b200 import abi as api
from blance_b200 import tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "blance_plan_chains_exposure"


# ---- ABI --------------------------------------------------------------------------------------------------------

def test_declaration_matches_header():
    probe = r'''
    #include <stddef.h>
    #include <stdio.h>
    #include "blance_b200.h"
    typedef int (*fn)(blance_ctx*, const blance_plan_in*, int32_t, int32_t, const blance_chain_stage*, const blance_scenario_opts*,
                      int32_t, int32_t, int32_t, const int32_t*, const uint8_t*, blance_scenario_out*, blance_chain_out*,
                      blance_scenario_schedule_out*, const blance_audit_opts*, blance_audit_out*, const blance_audit_opts*,
                      int32_t, blance_exposure_out*, blance_scenario_schedule_out*, blance_exposure_out*, blance_chain_span_out*);
    int main(void) {
    #ifdef CHECK
      fn f = blance_plan_chains_exposure; (void)f;
    #endif
      printf("%zu %zu %zu %zu\n", sizeof(blance_chain_span_out), offsetof(blance_chain_span_out, peak),
             offsetof(blance_chain_span_out, part_min_copies), offsetof(blance_chain_span_out, dom_peak_round));
      return 0;
    }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        inc = ["-I", os.path.join(ROOT, "include")]
        # -Werror: a prototype that differs from the typedef in any argument does not compile
        subprocess.run(["gcc", "-Werror", "-Wincompatible-pointer-types", "-DCHECK"] + inc + [c, "-c", "-o", os.path.join(d, "p.o")], check=True)
        subprocess.run(["gcc"] + inc + [c, "-o", os.path.join(d, "p")], check=True)
        sizes = [int(x) for x in subprocess.run([os.path.join(d, "p")], stdout=subprocess.PIPE, text=True, check=True).stdout.split()]
    S = api.ChainSpanOut
    assert sizes == [ctypes.sizeof(S), S.peak.offset, S.part_min_copies.offset, S.dom_peak_round.offset]
    lib = api.capi()
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    assert lib.blance_plan_chains_exposure.argtypes == [vp, vp, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp,
                                                        vp, vp, vp]
    assert NAME in api.EXPORTS


# ---- argument errors without a device ---------------------------------------------------------------------------

def _null_ctx():
    c = tables.Context.__new__(tables.Context)
    c.lib, c.ptr, c._rounds = api.capi(), ctypes.c_void_p(), {}
    return c


def _small(T=2):
    t, rng = random_base(3)
    return t, random_chains(t, rng, 2, T)


def _raw(t, T=2, n_move_conc=1, net=True, expo=True, net_sched=False, net_expo=False, span=None, series_cap=0, eopts=None,
         n_parts=None, n_slots=None, dom=False, node_in_all=1):
    """blance_plan_chains_exposure with ctx NULL, one chain of T stages without node changes, raw arguments.  span:
    None, or the name of one span array to ask for."""
    lib = api.capi()
    base = t.struct()
    if n_parts is not None:
        base.n_parts, base.n_slots = n_parts, n_slots
    inall = np.full(max(1, t.n_nodes), node_in_all, np.uint8)
    sts = (api.ChainStage * T)()
    for s in range(T):
        sts[s].nodes.node_removed, sts[s].nodes.node_added = base.node_removed, base.node_added
        sts[s].node_in_all = inall.ctypes.data
    nc = max(1, n_move_conc)
    out = (api.ScenarioOut * T)()
    sched = (api.ScenarioScheduleOut * (T * nc))()
    counts = (ctypes.c_int32 * nc)(*([1] * nc))
    buf = np.zeros(max(1, t.n_node_ids, t.n_parts), np.int64)
    ex = (api.ExposureOut * (T * nc))()
    if dom:
        ex[T * nc - 1].dom_peak = buf.ctypes.data
    sp = None
    if span is not None:
        sp = (api.ChainSpanOut * nc)()
        setattr(sp[0], span, buf.ctypes.data)
    st = lib.blance_plan_chains_exposure(None, ctypes.byref(base), 1, T, sts, None, 0, 0, n_move_conc, counts if n_move_conc else None,
                                         None, out, (api.ChainOut * 1)() if net else None, sched, None, None,
                                         None if eopts is None else ctypes.byref(eopts), series_cap, ex if expo else None,
                                         (api.ScenarioScheduleOut * nc)() if net_sched else None,
                                         (api.ExposureOut * nc)() if net_expo else None, sp)
    return st, lib.blance_last_error(None).decode()


def test_errors_with_a_null_context():
    t, _ = _small()
    st, msg = _raw(t, n_move_conc=0)
    assert st == -1 and NAME in msg and "n_move_conc" in msg
    st, msg = _raw(t, series_cap=-1)
    assert st == -1 and "series_cap" in msg
    st, msg = _raw(t, net=False, net_sched=True)
    assert st == -1 and "need net" in msg
    st, msg = _raw(t, net=False, net_expo=True)
    assert st == -1 and "need net" in msg
    st, msg = _raw(t, expo=False, net_expo=True)
    assert st == -1 and "need expo" in msg
    for f in ("part_min_copies", "part_no_top", "part_flags", "dom_peak", "dom_peak_stage", "dom_peak_round"):
        st, msg = _raw(t, expo=False, span=f)
        assert st == -1 and "need expo" in msg, f
    st, msg = _raw(t, eopts=api.AuditOpts(api.AUDIT_N2N, 0, None))
    assert st == -1 and "eopts.flags" in msg
    cyc = np.arange(t.n_node_ids + 1, dtype=np.int32)
    cyc[:t.n_node_ids] = t.n_node_ids
    st, msg = _raw(t, eopts=api.AuditOpts(0, 1, cyc.ctypes.data))
    assert st == -1 and "cycle" in msg
    # everything blance_plan_chains rejects, named by chain and stage
    st, msg = _raw(t, T=0)
    assert st == -1 and "n_stages" in msg
    st, msg = _raw(t, node_in_all=3)
    assert st == -1 and "chain 0, stage 0: node_in_all" in msg
    # every argument passes (the schedule's arrays only, the span's schedule arrays): the NULL context stops the call
    for span in (None, "node_last_round", "part_done_round"):
        st, msg = _raw(t, expo=False, span=span, net_sched=True)
        assert st == -1 and msg == "ctx is NULL", (span, msg)
    st, msg = _raw(t, net_sched=True, net_expo=True, span="dom_peak", series_cap=3)
    assert st == -1 and msg == "ctx is NULL", msg


EVENTS_FIT, EVENTS_OVER = (1 << 31) // 68, (1 << 31) // 68 + 1


@pytest.mark.parametrize("where", ["stage", "span"])
def test_static_event_bound_at_the_edge(where):
    t, _ = _small()
    kw = dict(stage=dict(dom=True), span=dict(span="dom_peak_round"))[where]
    st, msg = _raw(t, n_parts=EVENTS_OVER, n_slots=1, **kw)
    assert st == -2 and "2^31" in msg, msg
    assert ("chain 0, stage 1, count 0" in msg) if where == "stage" else ("span" in msg)
    st, msg = _raw(t, n_parts=EVENTS_FIT, n_slots=1, **kw)
    assert st != -2 and "2^31" not in msg, msg


def test_python_wrapper_errors():
    c = _null_ctx()
    t, chains = _small()
    for kw in (dict(exposure={}), dict(audit={}), dict(span=True), dict(node_has_mover=np.ones(t.n_node_ids))):
        with pytest.raises(ValueError, match="need a schedule"):
            c.plan_chains(t, chains, False, **kw)
    with pytest.raises(ValueError, match="at least one count"):
        c.plan_chains(t, chains, False, schedule=[])
    with pytest.raises(KeyError, match="serie_cap"):
        c.plan_chains(t, chains, False, schedule=[1], exposure=dict(serie_cap=3))
    with pytest.raises(ValueError, match="node_has_mover"):
        c.plan_chains(t, chains, False, schedule=[1], node_has_mover=np.ones(t.n_node_ids + 1))
    with pytest.raises(api.BlanceError, match="series_cap"):
        c.plan_chains(t, chains, False, schedule=[1], exposure=dict(series_cap=-2))
    with pytest.raises(api.BlanceError, match="ctx is NULL"):
        c.plan_chains(t, chains, True, schedule=[1, 2], audit={}, exposure=dict(series_cap=4), span=True)


# ---- the CPU reference against a literal replay -----------------------------------------------------------------

def _literal(t, next_rows, favor, count):
    """A stage's schedule read literally: the Go reading of OrchestrateSchedule's batches.  The stage's next rows come
    from chain_util.chain_reference, whose chain loop test_chains.py checks against the literal Go chain loop on
    string maps; here only the schedule and the exposure are replayed."""
    member, beg, end = REF.begmap_rows(t, next_rows)
    slot_off = np.asarray(t.state_slot_off, np.int32)
    off, node, state, kind = calc_moves(slot_off, beg, end, favor)
    mover = (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8)
    rounds = SO.go_reading(off, node, kind, t.n_node_ids, count, mover)
    s = go_summaries(off, node, t.n_node_ids, rounds)
    full = np.zeros(t.n_parts, np.int32)
    full[member] = s["part_done_round"]
    s["part_done_round"] = full
    return s


@pytest.mark.parametrize("seed", [1, 4, 12, 30])
def test_reference_equals_the_literal_replay(seed):
    t, rng = random_base(seed)
    opts = None
    if seed % 2:
        t = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
        opts = [dict(state_constraints=np.asarray(t.state_constraints, np.int32) + 1), {}]
    chains = random_chains(t, rng, 2, 3)
    parent = random_forest(rng, t.n_node_ids, 3) if seed % 3 else None
    counts = (1, 3)
    for i, chain in enumerate(chains):
        o = None if opts is None else opts[i]
        for favor in (False, True):
            stages, net, spans = CA.chain_analysis(t, chain, o, favor, counts, domain_parent=parent)
            lit, _, _ = CA.chain_analysis(t, chain, o, favor, counts, domain_parent=parent, oracle=EO.replay)
            ref, _ = C.chain_reference(t, chain, o, favor)
            cur = t
            for s, stage in enumerate(chain):
                x = C.substituted(cur, stage, o, s)
                for k, c in enumerate(counts):
                    assert_same_summaries(stages[s][k][0], _literal(x, ref[s]["next_rows"], favor, c), (seed, i, s, c))
                    EO.assert_equal(stages[s][k][1], lit[s][k][1], (seed, i, s, c))
                cur = C.advance(cur, ref[s]["next_rows"], ref[s]["next_shape"])
            for k in range(len(counts)):
                sp = spans[k]
                assert sp["rounds"] == sum(st[k][0]["rounds"] for st in stages)
                assert sp["peak"].tolist() == np.max([st[k][1]["peak"] for st in stages], axis=0).tolist()
                # a partition's span rounds lie inside the chain's
                assert (sp["part_done_round"] <= sp["rounds"]).all() and (sp["node_last_round"] <= sp["rounds"]).all()


def test_fold_by_hand():
    """Two stages of two partitions and two nodes: the G_t offsets, the last-stage rules and the first-stage ties."""
    s0 = dict(rounds=3, moves_done=4, stuck_parts=0, max_batch=2, node_rounds=np.array([2, 1], np.int32),
              node_last_round=np.array([3, 0], np.int32), part_done_round=np.array([2, 3], np.int32))
    s1 = dict(rounds=2, moves_done=1, stuck_parts=1, max_batch=1, node_rounds=np.array([0, 1], np.int32),
              node_last_round=np.array([0, 2], np.int32), part_done_round=np.array([0, -1], np.int32))
    e0 = dict(peak=np.array([1, 0, 2, 1, 0, 5]), peak_round=np.array([1, 0, 2, 1, 0, 0]), area=np.ones(6, np.int64),
              part_min_copies=np.array([1, -1], np.int32), part_no_top=np.array([1, 0], np.int32), part_flags=np.array([1, 0], np.uint8),
              dom_peak=np.array([2, 3]), dom_peak_round=np.array([1, 0], np.int32))
    e1 = dict(peak=np.array([1, 1, 3, 0, 0, 5]), peak_round=np.array([0, 2, 1, 0, 0, 1]), area=np.ones(6, np.int64),
              part_min_copies=np.array([2, 0], np.int32), part_no_top=np.array([2, 0], np.int32), part_flags=np.array([2, 8], np.uint8),
              dom_peak=np.array([2, 4]), dom_peak_round=np.array([2, 1], np.int32))
    sp = CA.fold([s0, s1], [e0, e1])
    assert (sp["rounds"], sp["moves_done"], sp["stuck_parts"], sp["max_batch"]) == (5, 5, 1, 2)
    assert sp["node_rounds"].tolist() == [2, 2] and sp["node_last_round"].tolist() == [3, 5]
    assert sp["part_done_round"].tolist() == [2, -1]
    assert sp["peak"].tolist() == [1, 1, 3, 1, 0, 5] and sp["peak_stage"].tolist() == [0, 1, 1, 0, 0, 0]
    assert sp["peak_round"].tolist() == [1, 2, 1, 1, 0, 0] and sp["area"].tolist() == [2] * 6
    assert sp["part_min_copies"].tolist() == [1, 0] and sp["part_no_top"].tolist() == [3, 0] and sp["part_flags"].tolist() == [3, 8]
    assert sp["dom_peak"].tolist() == [2, 4] and sp["dom_peak_stage"].tolist() == [0, 1] and sp["dom_peak_round"].tolist() == [1, 1]
