"""The argument checks of blance_map_audit and blance_plan_scenarios_audit: every one is made before any device work,
so they are observable without a device (and without a context); then a machine without a device gets
BLANCE_ERR_CUDA, never a result."""
import ctypes

import numpy as np
import pytest

from blance_b200 import api, tables

INVALID, UNSUPPORTED, CUDA = -1, -2, -3


def _have_gpu():
    ctx = ctypes.c_void_p()
    st = api.capi().blance_ctx_create(ctypes.byref(ctx), -1)
    if st == 0:
        api.capi().blance_ctx_destroy(ctx)
    return st == 0


def instance():
    t = tables.PlanTables(6, 2, 4, [0, 1], [1, 2])
    t.cur_shape[:] = 2
    t.cur_rows[:] = [0, 1, 2]
    return t


def call(t, opts=None, out=True, rows=True, shape=True, model=True):
    lib = api.capi()
    s = t.struct()
    r = tables.AuditResult(t, int(t.n_rules) if t.has_hier_rules else 0)
    st = lib.blance_map_audit(None, ctypes.byref(s) if model else None, t.cur_rows.ctypes.data if rows else None,
                              t.cur_shape.ctypes.data if shape else None, None if opts is None else ctypes.byref(opts),
                              ctypes.byref(r.out) if out else None)
    return st, lib.blance_last_error(None).decode()


def opts_of(parent=None, n_domains=None, flags=0):
    o = api.AuditOpts()
    o.flags = flags
    keep = None
    if parent is not None:
        keep = np.ascontiguousarray(parent, np.int32)
        o.domain_parent = keep.ctypes.data
    o.n_domains = n_domains if n_domains is not None else (0 if parent is None else len(parent) - 6)
    o._keep = keep
    return o


def test_null_arguments():
    t = instance()
    assert call(t, model=False)[0] == INVALID
    for kw in (dict(out=False), dict(rows=False), dict(shape=False)):
        st, msg = call(t, **kw)
        assert st == INVALID and "NULL" in msg, (kw, msg)


def test_bad_forests():
    t = instance()
    ok = [6, 6, 6, 7, 7, 7, 8, 8, -1]
    for parent, what in ((ok[:8] + [6], "cycle"), ([6, 6, 6, 7, 7, 7, 9, 8, -1], "outside"), ([-2] + ok[1:], "outside")):
        st, msg = call(t, opts_of(parent))
        assert st == INVALID and what in msg, (parent, msg)
    deep = [6] * 6 + list(range(7, 7 + 17)) + [-1]          # node -> 18 inner vertices in a chain: 18 edges
    st, msg = call(t, opts_of(deep))
    assert st == INVALID and "16 edges" in msg
    assert call(t, opts_of(None, n_domains=3))[0] == INVALID
    assert call(t, opts_of(ok, n_domains=-1))[0] == INVALID
    assert call(t, opts_of(flags=2))[0] == INVALID


def test_hierarchy_limits():
    t = instance()
    t.has_hier_rules, t.n_rules, t.n_hier_bits = 1, 1, 4097
    t.rule_off = np.array([0, 0, 1], np.int32)
    t.ie_mask = np.zeros(7 * 129, np.uint32)
    st, msg = call(t)
    assert st == UNSUPPORTED and "4096" in msg
    t.n_hier_bits = 6
    t.rule_off = np.array([0, 2, 1], np.int32)
    assert call(t)[0] == INVALID
    t.rule_off = np.array([0, 0, 1], np.int32)
    t.n_rules = 257
    assert call(t)[0] == UNSUPPORTED


def test_scenarios_audit_checks_its_arguments_first():
    t = instance()
    lib = api.capi()
    base = t.struct()
    scs = (api.Scenario * 1)()
    outs = (api.ScenarioOut * 1)()
    aud = (api.AuditOut * 1)()
    bad = opts_of([6] * 9)
    args = (None, ctypes.byref(base), 1, scs, None, 0, 0, 0, None, None, outs, None)
    assert lib.blance_plan_scenarios_audit(*args, None, None) == INVALID                  # no audit output
    assert lib.blance_plan_scenarios_audit(*args, ctypes.byref(bad), aud) == INVALID      # a cycle
    counts = (ctypes.c_int32 * 1)(1)
    assert lib.blance_plan_scenarios_audit(None, ctypes.byref(base), 1, scs, None, 0, 0, 1, counts, None, outs, None, None, aud) == INVALID


def test_no_device_is_an_error_not_a_result():
    if _have_gpu():
        pytest.skip("a CUDA device is present")
    t = instance()
    st, msg = call(t, opts_of([6, 6, 6, 7, 7, 7, 8, 8, -1], flags=api.AUDIT_N2N))
    assert st == CUDA and "no CPU fallback" in msg
    lib = api.capi()
    base = t.struct()
    scs, outs, aud = (api.Scenario * 1)(), (api.ScenarioOut * 1)(), (api.AuditOut * 1)()
    scs[0].node_removed = scs[0].node_added = t.node_removed.ctypes.data
    assert lib.blance_plan_scenarios_audit(None, ctypes.byref(base), 1, scs, None, 0, 0, 0, None, None, outs, None, None, aud) == CUDA
