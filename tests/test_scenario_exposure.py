"""blance_plan_scenarios_exposure (include/blance_b200.h), CPU side: the ctypes declaration against the header, every
argument error with a NULL context (no device needed), the Python wrapper's own errors, and the CPU reference of the
wave semantics (tests/scenario_exposure_ref.py: the CPU plan, its begMap moves, the schedule oracle, the vectorised
exposure oracle) against the literal replay on random bases with options, prev-only partitions and partitions in
neither map."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import exposure_oracle as EO
import scenario_exposure_ref as REF
from test_exposure_oracle import random_forest
from test_scenarios_gpu import oracle_tables, random_base, random_scenarios

from blance_b200 import abi as api
from blance_b200 import tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "blance_plan_scenarios_exposure"


# ---- ABI --------------------------------------------------------------------------------------------------------

def test_declaration_matches_header():
    probe = r'''
    #include <stdio.h>
    #include "blance_b200.h"
    typedef int (*fn)(blance_ctx*, const blance_plan_in*, int32_t, const blance_scenario*, const blance_scenario_opts*,
                      int32_t, int32_t, int32_t, const int32_t*, const uint8_t*, blance_scenario_out*,
                      blance_scenario_schedule_out*, const blance_audit_opts*, blance_audit_out*, const blance_audit_opts*,
                      int32_t, blance_exposure_out*);
    int main(void) { fn f = blance_plan_scenarios_exposure; (void)f; printf("%zu\n", sizeof(blance_exposure_out)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        # -Werror: a prototype that differs from the typedef in any argument does not compile; only main is linked
        subprocess.run(["gcc", "-Werror", "-Wincompatible-pointer-types", "-I", os.path.join(ROOT, "include"), c, "-c", "-o",
                        os.path.join(d, "p.o")], check=True)
    lib = api.capi()
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    assert lib.blance_plan_scenarios_exposure.argtypes == [vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp]
    assert NAME in api.EXPORTS
    assert ctypes.sizeof(api.ExposureOut) == 184          # the struct is shared with blance_moves_exposure, unchanged


# ---- argument errors without a device ---------------------------------------------------------------------------

def _null_ctx():
    """A tables.Context whose blance_ctx* is NULL: every call reaches the library's argument checks only."""
    c = tables.Context.__new__(tables.Context)
    c.lib, c.ptr, c._rounds = api.capi(), ctypes.c_void_p(), {}
    return c


def _small():
    t, rng = random_base(3)
    return t, random_scenarios(t, rng, 2)


def _raw(t, n_move_conc=1, expo=True, series_cap=0, eopts=None, n_parts=None, n_slots=None, dom=False, aflags=None):
    """blance_plan_scenarios_exposure with ctx NULL, one base scenario (no node changes), raw arguments."""
    lib = api.capi()
    base = t.struct()
    if n_parts is not None:
        base.n_parts, base.n_slots = n_parts, n_slots
    sc = (api.Scenario * 1)()
    sc[0].node_removed, sc[0].node_added = base.node_removed, base.node_added
    out = (api.ScenarioOut * 1)()
    sched = (api.ScenarioScheduleOut * max(1, n_move_conc))()
    counts = (ctypes.c_int32 * max(1, n_move_conc))(*([1] * max(1, n_move_conc)))
    peaks = np.zeros(max(1, t.n_node_ids), np.int64)
    ex = (api.ExposureOut * max(1, n_move_conc))()
    if dom:
        ex[0].dom_peak = peaks.ctypes.data
    st = lib.blance_plan_scenarios_exposure(None, ctypes.byref(base), 1, sc, None, 0, 0, n_move_conc, counts if n_move_conc else None,
                                            None, out, sched, None if aflags is None else ctypes.byref(api.AuditOpts(aflags, 0, None)),
                                            None if aflags is None else (api.AuditOut * 1)(), None if eopts is None else ctypes.byref(eopts),
                                            series_cap, ex if expo else None)
    return st, lib.blance_last_error(None).decode()


def test_errors_with_a_null_context():
    t, _ = _small()
    st, msg = _raw(t, n_move_conc=0)
    assert st == -1 and NAME in msg and "n_move_conc" in msg
    st, msg = _raw(t, expo=False)
    assert st == -1 and "expo is NULL" in msg
    st, msg = _raw(t, series_cap=-1)
    assert st == -1 and "series_cap" in msg
    st, msg = _raw(t, eopts=api.AuditOpts(api.AUDIT_N2N, 0, None))
    assert st == -1 and "eopts.flags" in msg
    bad = np.full(t.n_node_ids, t.n_node_ids + 3, np.int32)
    st, msg = _raw(t, eopts=api.AuditOpts(0, 0, bad.ctypes.data))
    assert st == -1 and "domain_parent" in msg
    cyc = np.arange(t.n_node_ids + 1, dtype=np.int32)
    cyc[:t.n_node_ids] = t.n_node_ids
    st, msg = _raw(t, eopts=api.AuditOpts(0, 1, cyc.ctypes.data))
    assert st == -1 and "cycle" in msg
    # everything blance_plan_scenarios_audit rejects, named by scenario
    c = _null_ctx()
    base, scs = _small()
    scs[1]["add_is_nil"] = 7
    with pytest.raises(api.BlanceError, match="scenario 1: add_is_nil"):
        c.plan_scenarios(base, scs, False, schedule=[1], exposure={})
    base, scs = _small()
    st, msg = _raw(base, aflags=8)
    assert st == -1 and "audit flags" in msg
    # every argument passes: the NULL context is what stops the call
    with pytest.raises(api.BlanceError, match="ctx is NULL"):
        c.plan_scenarios(base, scs, False, schedule=[1, 2], exposure=dict(series_cap=4))


# 2 x 17 x 2 x n_slots x n_parts: the fault-domain events one instance may emit; with one slot, 68 x P crosses 2^31
# between these two partition counts (2^31 is no multiple of 17, so no count lands on it exactly)
EVENTS_FIT, EVENTS_OVER = (1 << 31) // 68, (1 << 31) // 68 + 1


def test_static_event_bound_at_the_edge():
    t, _ = _small()
    assert 68 * EVENTS_FIT < (1 << 31) <= 68 * EVENTS_OVER
    st, msg = _raw(t, n_parts=EVENTS_OVER, n_slots=1, dom=True)
    assert st == -2 and "scenario 0, count 0" in msg and "2^31" in msg, msg       # BLANCE_ERR_UNSUPPORTED
    st, msg = _raw(t, n_parts=EVENTS_FIT, n_slots=1, dom=True)
    assert st != -2 and "2^31" not in msg, msg      # past the bound check; a NULL context then stops it
    st, msg = _raw(t, n_parts=EVENTS_OVER, n_slots=1, dom=False)
    assert st != -2, msg                            # without dom peaks there is no event bound


def test_python_wrapper_errors():
    c = _null_ctx()
    t, scs = _small()
    with pytest.raises(ValueError, match="needs a schedule"):
        c.plan_scenarios(t, scs, False, exposure={})
    with pytest.raises(ValueError, match="needs a schedule"):
        c.plan_scenarios(t, scs, False, schedule=[], exposure={})
    with pytest.raises(KeyError, match="serie_cap"):
        c.plan_scenarios(t, scs, False, schedule=[1], exposure=dict(serie_cap=3))
    with pytest.raises(api.BlanceError, match="series_cap"):
        c.plan_scenarios(t, scs, False, schedule=[1], exposure=dict(series_cap=-2))


# ---- the CPU reference of the wave semantics --------------------------------------------------------------------

def _with_neither(t, rng):
    """Some partitions absent from both maps, some in prevMap only (not assigned)."""
    P = t.n_parts
    t.part_in_assign[:] = (rng.random(P) < 0.7).astype(np.uint8)
    gone = rng.random(P) < 0.1
    t.part_in_prev[gone] = 0
    t.part_in_assign[gone] = 0
    t.prev_rows.reshape(P, -1)[gone] = -1
    t.prev_shape.reshape(P, -1)[gone] = 0
    return t


@pytest.mark.parametrize("seed", [1, 4, 12, 30])
def test_reference_equals_the_literal_replay(seed):
    t, rng = random_base(seed)
    t = _with_neither(t, rng)
    opts = None
    if seed % 2:
        t = tables.widen_layout(t, [int(x) + 1 for x in t.state_constraints])
        opts = [{}, dict(state_constraints=np.asarray(t.state_constraints, np.int32) + 1)]
    scs = random_scenarios(t, rng, 2)
    for sc in scs:                           # plan.go:544: no removal with partitions absent from prevMap
        sc["node_removed"][:] = 0
    parent = random_forest(rng, t.n_node_ids, 3) if seed % 3 else None
    neither = (t.part_in_prev == 0) & (t.part_in_assign == 0)
    assert neither.any() and ((t.part_in_prev != 0) & (t.part_in_assign == 0)).any()
    for i, sc in enumerate(scs):
        st = tables.scenario_tables(t, sc, None if opts is None else opts[i])
        nxt = oracle_tables(st).next_rows
        for favor in (False, True):
            for count in (1, 3):
                got, sc_ = REF.scenario_exposure(st, nxt, favor, count, domain_parent=parent)
                lit, _ = REF.scenario_exposure(st, nxt, favor, count, domain_parent=parent, oracle=EO.replay)
                EO.assert_equal(got, lit, (seed, i, favor, count))
                assert (got["part_min_copies"][neither] == -1).all() and not got["part_no_top"][neither].any()
                assert not got["part_flags"][neither].any() and got["rounds"] == sc_["rounds"]
