"""Every scenario and chain entry point with a NULL context, row by row: one bad argument at a time, and a few rows
with two that pin which check fires first.  Each row pins the exact (status, message) and how many schedule outputs
the call cleared before it failed.  Rows whose result depends on whether the machine has a device (the audit entry's
NULL context) accept exactly its two outcomes."""
import ctypes

import numpy as np
import pytest

from blance_b200 import abi as api
from blance_b200 import tables

INVALID, UNSUPPORTED, CUDA = -1, -2, -3
NO_DEVICE = (CUDA, "no CUDA device available; libblance_b200 has no CPU fallback")
NULL_CTX = (INVALID, "ctx is NULL")
NEED_CTX = "need_ctx"              # NO_DEVICE without a device, NULL_CTX with one
EVENTS_OVER = (1 << 31) // 68 + 1  # n_parts of one slot just over 2 x 17 x 2 x n_slots x n_parts < 2^31
STALE = 99                         # the rounds every schedule output holds before the call


def _base():
    t = tables.PlanTables(4, 2, 6, [0, 1], [1, 1], n_node_ids=5)
    t.part_in_prev[:] = 1
    return t


class _Call:
    """The arguments of one call, valid unless a knob says otherwise.  Item 1 (scenario 1, or stage 1 of chain 1)
    carries the bad scenario or options, the last exposure, net exposure or span output the dom_peak asked for."""

    def __init__(self, chains, n=2, T=2, base=True, sc=True, out=True, scen=None, opts=None, nmc=2, mc=True, sched=True, aflags=0,
                 audit=True, eopts=None, series_cap=0, expo=True, dom=False, net=True, net_sched=False, net_expo=False,
                 net_dom=False, span=None, n_parts=None, max_iters=None, in_all=1):
        t = self.t = _base()
        if max_iters is not None:
            t.max_iters = max_iters
        b = self.base = t.struct()
        if n_parts is not None:
            b.n_parts, b.n_slots = n_parts, 1
        self.n, self.T, self.nmc = n, T, nmc
        m, nc, per = max(1, n), max(1, min(nmc, 8)), max(1, T) if chains else 1
        self.sc = (api.Scenario * m)()
        self.stages = (api.ChainStage * (m * max(1, T)))()
        self.in_all = np.full(t.n_nodes, in_all or 0, np.uint8)
        for x in range(m * max(1, T)):
            s = self.stages[x]
            s.nodes.node_removed, s.nodes.node_added = b.node_removed, b.node_added
            s.node_in_all = None if in_all is None else self.in_all.ctypes.data
        for i in range(m):
            self.sc[i].node_removed, self.sc[i].node_added = b.node_removed, b.node_added
        for k, v in (scen or {}).items():
            setattr(self.sc[min(1, m - 1)], k, v)
            setattr(self.stages[min(1, m - 1) * max(1, T) + min(1, max(1, T) - 1)].nodes, k, v)
        self.opts = None
        if opts is not None:
            self.opts = (api.ScenarioOpts * m)()
            for k, v in opts.items():
                setattr(self.opts[min(1, m - 1)], k, v)
        self.out = (api.ScenarioOut * (m * max(1, T)))() if out else None
        self.mc = (ctypes.c_int32 * max(1, nmc))(*([1] * max(1, nmc))) if mc else None
        self.sched = (api.ScenarioScheduleOut * (m * max(1, T) * nc))() if sched else None
        for x in range(m * max(1, T) * nc if sched else 0):
            self.sched[x].rounds = STALE
        self.aopts = api.AuditOpts(aflags, 0, None)
        self.audit = (api.AuditOut * (m * max(1, T)))() if audit else None
        self.eopts = eopts
        self.series_cap = series_cap
        self.buf = np.zeros(max(1, t.n_node_ids, t.n_parts), np.int64)
        self.expo = (api.ExposureOut * (m * max(1, T) * nc))() if expo else None
        if dom:
            self.expo[m * per * nc - 1].dom_peak = self.buf.ctypes.data
        self.net = (api.ChainOut * m)() if net else None
        self.net_sched = (api.ScenarioScheduleOut * (m * nc))() if net_sched else None
        self.net_expo = (api.ExposureOut * (m * nc))() if net_expo else None
        if net_dom:
            self.net_expo[m * nc - 1].dom_peak = self.buf.ctypes.data
        self.span = None
        if span is not None:
            self.span = (api.ChainSpanOut * (m * nc))()
            setattr(self.span[m * nc - 1], span, self.buf.ctypes.data)
        self.base_p = ctypes.byref(b) if base else None
        self.sc_p = self.sc if sc else None
        self.stages_p = self.stages if sc else None
        self.eopts_p = None if eopts is None else ctypes.byref(eopts)

    def cleared(self):
        if self.sched is None:
            return 0
        return sum(1 for s in self.sched if s.rounds == 0)


def _invoke(entry, c):
    lib = api.capi()
    if entry == "plain":
        return lib.blance_plan_scenarios(None, c.base_p, c.n, c.sc_p, 0, 0, c.out)
    if entry == "ex":
        return lib.blance_plan_scenarios_ex(None, c.base_p, c.n, c.sc_p, c.opts, 0, 0, c.out)
    if entry == "schedule":
        return lib.blance_plan_scenarios_schedule(None, c.base_p, c.n, c.sc_p, c.opts, 0, 0, c.nmc, c.mc, None, c.out, c.sched)
    if entry == "audit":
        return lib.blance_plan_scenarios_audit(None, c.base_p, c.n, c.sc_p, c.opts, 0, 0, c.nmc, c.mc, None, c.out, c.sched,
                                               ctypes.byref(c.aopts), c.audit)
    if entry == "exposure":
        return lib.blance_plan_scenarios_exposure(None, c.base_p, c.n, c.sc_p, c.opts, 0, 0, c.nmc, c.mc, None, c.out, c.sched,
                                                  ctypes.byref(c.aopts), c.audit, c.eopts_p, c.series_cap, c.expo)
    if entry == "chains":
        return lib.blance_plan_chains(None, c.base_p, c.n, c.T, c.stages_p, c.opts, 0, 0, c.out, c.net)
    assert entry == "chains_exposure"
    return lib.blance_plan_chains_exposure(None, c.base_p, c.n, c.T, c.stages_p, c.opts, 0, 0, c.nmc, c.mc, None, c.out, c.net,
                                           c.sched, ctypes.byref(c.aopts), c.audit, c.eopts_p, c.series_cap, c.expo,
                                           c.net_sched, c.net_expo, c.span)


def _cycle():
    p = np.arange(5 + 1, dtype=np.int32)
    p[:5] = 5
    _cycle.keep = p
    return api.AuditOpts(0, 1, p.ctypes.data)


BAD_SCEN = dict(scen=dict(add_is_nil=2))
BAD_OPTS = dict(opts=dict(set=0x100))
BAD_RULES = dict(opts=dict(set=api.OPT_HIERARCHY, has_hier_rules=1))     # rule_off NULL: the audit model check fires

# (entry, row name, knobs, (status, message) or NEED_CTX, schedule outputs cleared)
ROWS = [
    # each entry point: every argument valid, then one bad argument at a time
    ("plain", "ok", {},
     NULL_CTX, 0),
    ("plain", "n", dict(n=0),
     (INVALID, "blance_plan_scenarios: n must be positive"), 0),
    ("plain", "base", dict(base=False),
     (INVALID, "blance_plan_scenarios: base, sc or out is NULL"), 0),
    ("plain", "sc", dict(sc=False),
     (INVALID, "blance_plan_scenarios: base, sc or out is NULL"), 0),
    ("plain", "out", dict(out=False),
     (INVALID, "blance_plan_scenarios: base, sc or out is NULL"), 0),
    ("plain", "scenario", BAD_SCEN,
     (INVALID, "blance_plan_scenarios: scenario 1: add_is_nil is neither 0 nor 1"), 0),
    ("ex", "ok", {},
     NULL_CTX, 0),
    ("ex", "n", dict(n=-1),
     (INVALID, "blance_plan_scenarios_ex: n must be positive"), 0),
    ("ex", "base", dict(base=False),
     (INVALID, "blance_plan_scenarios_ex: base, sc or out is NULL"), 0),
    ("ex", "out", dict(out=False),
     (INVALID, "blance_plan_scenarios_ex: base, sc or out is NULL"), 0),
    ("ex", "scenario", BAD_SCEN,
     (INVALID, "blance_plan_scenarios_ex: scenario 1: add_is_nil is neither 0 nor 1"), 0),
    ("ex", "opts", BAD_OPTS,
     (INVALID, "blance_plan_scenarios_ex: scenario 1: opts.set has an unknown bit"), 0),
    # blance_plan_scenarios_schedule looks at the context before its arguments
    ("schedule", "ok", {},
     NULL_CTX, 0),
    ("schedule", "n", dict(n=0),
     NULL_CTX, 0),
    ("schedule", "base", dict(base=False),
     NULL_CTX, 0),
    ("schedule", "scenario", BAD_SCEN,
     NULL_CTX, 0),
    ("schedule", "n_move_conc", dict(nmc=0),
     NULL_CTX, 0),
    ("schedule", "sched", dict(sched=False),
     NULL_CTX, 0),
    # blance_plan_scenarios_audit reports a NULL context through need_ctx, after its own checks and before the scenarios'
    ("audit", "ok", {},
     NEED_CTX, 4),
    ("audit", "no schedule", dict(nmc=0, mc=False, sched=False),
     NEED_CTX, 0),
    ("audit", "n", dict(n=0),
     NEED_CTX, 0),
    ("audit", "base", dict(base=False),
     (INVALID, "blance_plan_scenarios_audit: base is NULL"), 0),
    ("audit", "sc", dict(sc=False),
     NEED_CTX, 0),
    ("audit", "out", dict(out=False),
     NEED_CTX, 0),
    ("audit", "scenario", BAD_SCEN,
     NEED_CTX, 4),
    ("audit", "opts", BAD_OPTS,
     NEED_CTX, 4),
    ("audit", "n_move_conc", dict(nmc=0),
     (INVALID, "blance_plan_scenarios_audit: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("audit", "sched", dict(sched=False),
     (INVALID, "blance_plan_scenarios_audit: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("audit", "2^29", dict(n_parts=1 << 29),
     (UNSUPPORTED, "blance_plan_scenarios_audit: 2^29 or more partitions"), 0),
    ("audit", "audit out", dict(audit=False),
     (INVALID, "blance_plan_scenarios_audit: the audit output is NULL"), 0),
    ("audit", "audit flags", dict(aflags=0x80),
     (INVALID, "blance_plan_scenarios_audit: audit flags hold an unknown bit"), 0),
    ("audit", "audit model", BAD_RULES,
     (INVALID, "blance_plan_scenarios_audit: scenario 1: rule_off is NULL"), 4),
    ("exposure", "ok", {},
     NULL_CTX, 4),
    ("exposure", "no audit", dict(audit=False),
     NULL_CTX, 4),
    ("exposure", "n", dict(n=0),
     (INVALID, "blance_plan_scenarios_exposure: n must be positive"), 0),
    ("exposure", "base", dict(base=False),
     (INVALID, "blance_plan_scenarios_exposure: base is NULL"), 0),
    ("exposure", "sc", dict(sc=False),
     (INVALID, "blance_plan_scenarios_exposure: base, sc or out is NULL"), 0),
    ("exposure", "out", dict(out=False),
     (INVALID, "blance_plan_scenarios_exposure: base, sc or out is NULL"), 0),
    ("exposure", "scenario", BAD_SCEN,
     (INVALID, "blance_plan_scenarios_exposure: scenario 1: add_is_nil is neither 0 nor 1"), 4),
    ("exposure", "opts", BAD_OPTS,
     (INVALID, "blance_plan_scenarios_exposure: scenario 1: opts.set has an unknown bit"), 4),
    ("exposure", "n_move_conc", dict(nmc=0),
     (INVALID, "blance_plan_scenarios_exposure: an exposure needs a schedule: n_move_conc must be positive"), 0),
    ("exposure", "move_conc", dict(mc=False),
     (INVALID, "blance_plan_scenarios_exposure: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("exposure", "2^29", dict(n_parts=1 << 29, audit=False),
     (UNSUPPORTED, "blance_plan_scenarios_exposure: 2^29 or more partitions"), 0),
    ("exposure", "nc x parts", dict(n_parts=1 << 20, nmc=1 << 12, audit=False),
     (UNSUPPORTED, "blance_plan_scenarios_exposure: n_move_conc x n_parts exceeds 2^31 - 1"), 0),
    ("exposure", "audit flags", dict(aflags=0x80),
     (INVALID, "blance_plan_scenarios_exposure: audit flags hold an unknown bit"), 0),
    # without an audit output the audit model is not checked: the event bound, checked after it, fires instead
    ("exposure", "no audit model check without audit", dict(BAD_RULES, audit=False, dom=True, n_parts=EVENTS_OVER),
     (UNSUPPORTED, "blance_plan_scenarios_exposure: scenario 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 4),
    ("exposure", "audit model", BAD_RULES,
     (INVALID, "blance_plan_scenarios_exposure: scenario 1: rule_off is NULL"), 4),
    ("exposure", "expo", dict(expo=False),
     (INVALID, "blance_plan_scenarios_exposure: expo is NULL"), 4),
    ("exposure", "series_cap", dict(series_cap=-1),
     (INVALID, "blance_plan_scenarios_exposure: series_cap is negative"), 4),
    ("exposure", "eopts.flags", dict(eopts=api.AuditOpts(1, 0, None)),
     (INVALID, "blance_plan_scenarios_exposure: eopts.flags must be 0 (eopts carries a forest only)"), 4),
    ("exposure", "eopts forest", dict(eopts="cycle"),
     (INVALID, "blance_plan_scenarios_exposure: domain_parent has a cycle or a vertex more than 16 edges below its root (vertex 0)"), 4),
    ("exposure", "event bound", dict(dom=True, n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_scenarios_exposure: scenario 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 4),
    ("exposure", "event bound fits", dict(dom=True, n_parts=EVENTS_OVER - 1, audit=False),
     (INVALID, "blance_plan_scenarios_exposure: scenario 0: state_slot_off[S] != n_slots"), 4),
    ("chains", "ok", {},
     NULL_CTX, 0),
    ("chains", "n", dict(n=0),
     (INVALID, "blance_plan_chains: n must be positive"), 0),
    ("chains", "n_stages", dict(T=0),
     (INVALID, "blance_plan_chains: n_stages must be positive"), 0),
    ("chains", "base", dict(base=False),
     (INVALID, "blance_plan_chains: base, stages or out is NULL"), 0),
    ("chains", "stages", dict(sc=False),
     (INVALID, "blance_plan_chains: base, stages or out is NULL"), 0),
    ("chains", "out", dict(out=False),
     (INVALID, "blance_plan_chains: base, stages or out is NULL"), 0),
    ("chains", "max_iters", dict(max_iters=0),
     (INVALID, "blance_plan_chains: a chain of several stages needs max_iters >= 1"), 0),
    ("chains", "max_iters one stage", dict(max_iters=0, T=1),
     NULL_CTX, 0),
    ("chains", "stage", BAD_SCEN,
     (INVALID, "blance_plan_chains: chain 1, stage 1: add_is_nil is neither 0 nor 1"), 0),
    ("chains", "opts", BAD_OPTS,
     (INVALID, "blance_plan_chains: chain 1, stage 0: opts.set has an unknown bit"), 0),
    ("chains", "node_in_all", dict(in_all=3),
     (INVALID, "blance_plan_chains: chain 0, stage 0: node_in_all is neither 0 nor 1"), 0),
    ("chains", "node_in_all NULL", dict(in_all=None),
     (INVALID, "blance_plan_chains: chain 0, stage 0: node_in_all is NULL"), 0),
    ("chains_exposure", "ok", {},
     NULL_CTX, 8),
    ("chains_exposure", "everything", dict(net_sched=True, net_expo=True, span="dom_peak", series_cap=3),
     NULL_CTX, 8),
    ("chains_exposure", "n", dict(n=0),
     (INVALID, "blance_plan_chains_exposure: n must be positive"), 0),
    ("chains_exposure", "n_stages", dict(T=0),
     (INVALID, "blance_plan_chains_exposure: n_stages must be positive"), 0),
    ("chains_exposure", "base", dict(base=False),
     (INVALID, "blance_plan_chains_exposure: base, stages or out is NULL"), 0),
    ("chains_exposure", "stages", dict(sc=False),
     (INVALID, "blance_plan_chains_exposure: base, stages or out is NULL"), 8),
    ("chains_exposure", "out", dict(out=False),
     (INVALID, "blance_plan_chains_exposure: base, stages or out is NULL"), 8),
    ("chains_exposure", "max_iters", dict(max_iters=0),
     (INVALID, "blance_plan_chains_exposure: a chain of several stages needs max_iters >= 1"), 8),
    ("chains_exposure", "stage", BAD_SCEN,
     (INVALID, "blance_plan_chains_exposure: chain 1, stage 1: add_is_nil is neither 0 nor 1"), 8),
    ("chains_exposure", "opts", BAD_OPTS,
     (INVALID, "blance_plan_chains_exposure: chain 1, stage 0: opts.set has an unknown bit"), 8),
    ("chains_exposure", "node_in_all", dict(in_all=3),
     (INVALID, "blance_plan_chains_exposure: chain 0, stage 0: node_in_all is neither 0 nor 1"), 8),
    ("chains_exposure", "n_move_conc", dict(nmc=0),
     (INVALID, "blance_plan_chains_exposure: n_move_conc must be positive"), 0),
    ("chains_exposure", "move_conc", dict(mc=False),
     (INVALID, "blance_plan_chains_exposure: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("chains_exposure", "sched", dict(sched=False),
     (INVALID, "blance_plan_chains_exposure: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("chains_exposure", "2^29", dict(n_parts=1 << 29, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: 2^29 or more partitions"), 0),
    ("chains_exposure", "net_sched", dict(net=False, net_sched=True),
     (INVALID, "blance_plan_chains_exposure: net_sched and net_expo need net"), 0),
    ("chains_exposure", "net_expo", dict(net=False, net_expo=True),
     (INVALID, "blance_plan_chains_exposure: net_sched and net_expo need net"), 0),
    ("chains_exposure", "net_expo without expo", dict(expo=False, net_expo=True),
     (INVALID, "blance_plan_chains_exposure: net_expo and the span's exposure arrays need expo"), 8),
    ("chains_exposure", "span without expo", dict(expo=False, span="part_flags"),
     (INVALID, "blance_plan_chains_exposure: net_expo and the span's exposure arrays need expo"), 8),
    ("chains_exposure", "span schedule only", dict(expo=False, span="part_done_round"),
     NULL_CTX, 8),
    ("chains_exposure", "audit flags", dict(aflags=0x80),
     (INVALID, "blance_plan_chains_exposure: audit flags hold an unknown bit"), 0),
    ("chains_exposure", "audit model", BAD_RULES,
     (INVALID, "blance_plan_chains_exposure: chain 1: rule_off is NULL"), 0),
    ("chains_exposure", "series_cap", dict(series_cap=-1),
     (INVALID, "blance_plan_chains_exposure: series_cap is negative"), 8),
    ("chains_exposure", "eopts.flags", dict(eopts=api.AuditOpts(1, 0, None)),
     (INVALID, "blance_plan_chains_exposure: eopts.flags must be 0 (eopts carries a forest only)"), 8),
    ("chains_exposure", "eopts forest", dict(eopts="cycle"),
     (INVALID, "blance_plan_chains_exposure: domain_parent has a cycle or a vertex more than 16 edges below its root (vertex 0)"), 8),
    ("chains_exposure", "event bound", dict(dom=True, n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: chain 1, stage 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    ("chains_exposure", "net event bound", dict(net_expo=True, net_dom=True, n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: chain 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    ("chains_exposure", "span event bound", dict(span="dom_peak_stage", n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: span: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    # two bad arguments: which check fires first
    ("audit", "base before audit out", dict(base=False, audit=False),
     (INVALID, "blance_plan_scenarios_audit: base is NULL"), 0),
    ("audit", "n_move_conc before scenario", dict(nmc=0, **BAD_SCEN),
     (INVALID, "blance_plan_scenarios_audit: n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("audit", "audit model before scenario", dict(BAD_RULES, scen=dict(add_is_nil=2)),
     (INVALID, "blance_plan_scenarios_audit: scenario 1: rule_off is NULL"), 4),
    ("exposure", "audit before n_move_conc", dict(aflags=0x80, nmc=0),
     (INVALID, "blance_plan_scenarios_exposure: audit flags hold an unknown bit"), 0),
    ("exposure", "n_move_conc before series_cap", dict(nmc=0, series_cap=-1),
     (INVALID, "blance_plan_scenarios_exposure: an exposure needs a schedule: n_move_conc must be positive"), 0),
    ("exposure", "eopts before audit model", dict(BAD_RULES, eopts=api.AuditOpts(1, 0, None)),
     (INVALID, "blance_plan_scenarios_exposure: eopts.flags must be 0 (eopts carries a forest only)"), 4),
    ("exposure", "event bound before scenario", dict(dom=True, n_parts=EVENTS_OVER, scen=dict(add_is_nil=2), audit=False),
     (UNSUPPORTED, "blance_plan_scenarios_exposure: scenario 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 4),
    ("chains", "n before stages", dict(n=0, sc=False),
     (INVALID, "blance_plan_chains: n must be positive"), 0),
    ("chains_exposure", "net before audit", dict(net=False, net_sched=True, aflags=0x80),
     (INVALID, "blance_plan_chains_exposure: net_sched and net_expo need net"), 0),
    ("chains_exposure", "series_cap before n_stages", dict(T=0, series_cap=-1),
     (INVALID, "blance_plan_chains_exposure: series_cap is negative"), 0),
    ("chains_exposure", "n_move_conc before stages", dict(nmc=0, sc=False),
     (INVALID, "blance_plan_chains_exposure: n_move_conc must be positive"), 0),
    ("chains_exposure", "event bound before stage", dict(dom=True, n_parts=EVENTS_OVER, **BAD_SCEN, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: chain 1, stage 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    ("exposure", "n_move_conc before expo", dict(nmc=0, expo=False),
     (INVALID, "blance_plan_scenarios_exposure: an exposure needs a schedule: n_move_conc must be positive"), 0),
    ("exposure", "expo before audit model", dict(BAD_RULES, expo=False),
     (INVALID, "blance_plan_scenarios_exposure: expo is NULL"), 4),
    ("exposure", "audit model before event bound", dict(BAD_RULES, dom=True, n_parts=EVENTS_OVER),
     (INVALID, "blance_plan_scenarios_exposure: scenario 0: state_slot_off does not span [0, n_slots]"), 4),
    ("chains_exposure", "base before net", dict(base=False, net=False, net_sched=True),
     (INVALID, "blance_plan_chains_exposure: base, stages or out is NULL"), 0),
    ("chains_exposure", "audit model before n_move_conc", dict(BAD_RULES, nmc=0),
     (INVALID, "blance_plan_chains_exposure: chain 1: rule_off is NULL"), 0),
    ("chains_exposure", "series_cap before span without expo", dict(expo=False, span="part_flags", series_cap=-1),
     (INVALID, "blance_plan_chains_exposure: series_cap is negative"), 8),
    ("chains_exposure", "event bound before net event bound", dict(dom=True, net_expo=True, net_dom=True, n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: chain 1, stage 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    ("chains_exposure", "net event bound before span event bound",
     dict(net_expo=True, net_dom=True, span="dom_peak_stage", n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, "blance_plan_chains_exposure: chain 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
]


def run_row(entry, knobs):
    kw = dict(knobs)
    if kw.get("eopts") == "cycle":
        kw["eopts"] = _cycle()
    c = _Call(entry.startswith("chains"), **kw)
    st = _invoke(entry, c)
    return st, api.capi().blance_last_error(None).decode(), c.cleared()


@pytest.mark.parametrize("entry,name,knobs,want,cleared", ROWS, ids=["%s-%s" % (r[0], r[1]) for r in ROWS])
def test_null_context_row(entry, name, knobs, want, cleared):
    st, msg, n_cleared = run_row(entry, knobs)
    if want == NEED_CTX:
        assert (st, msg) in (NO_DEVICE, NULL_CTX)
    else:
        assert (st, msg) == want
    assert n_cleared == cleared
