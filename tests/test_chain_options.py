"""Chains whose stages set plan options of their own (blance_plan_chains_ex), CPU side: the ctypes declaration against
the header, every argument error with a NULL context (one row per option group and bad value, each naming the chain
and stage), and the per-stage chain reference (tests/chain_stage_util.py) against the literal oracle driven as the Go
loop with per-stage options on string maps.  The device path is tests/test_chain_options_gpu.py."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import chain_stage_util as CS
import golden_util as G
from randgen import random_instance
from test_chains import make_chain, unintern
from test_scenarios import removal_allowed
from test_wave_requests import BAD_SCEN, EVENTS_OVER, INVALID, NULL_CTX, UNSUPPORTED, _Call, _cycle

import blance_b200
from blance_b200 import abi as api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "blance_plan_chains_ex"
COUNT_BOUND = "sum of |partition weight| x slots plus the largest non-model count exceeds int32 (the device keeps int32 counts)"


# ---- ABI --------------------------------------------------------------------------------------------------------

def test_declaration_matches_header():
    probe = r'''
    #include "blance_b200.h"
    typedef int (*fn)(blance_ctx*, const blance_plan_in*, int32_t, int32_t, const blance_chain_stage*, const blance_scenario_opts*,
                      int32_t, int32_t, int32_t, const int32_t*, const uint8_t*, blance_scenario_out*, blance_chain_out*,
                      blance_scenario_schedule_out*, const blance_audit_opts*, blance_audit_out*, const blance_audit_opts*,
                      int32_t, blance_exposure_out*, blance_scenario_schedule_out*, blance_exposure_out*, blance_chain_span_out*);
    int main(void) { fn f = blance_plan_chains_ex; (void)f; return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        # -Werror: a prototype that differs from the typedef in any argument does not compile
        subprocess.run(["gcc", "-Werror", "-Wincompatible-pointer-types", "-I", os.path.join(ROOT, "include"), c, "-c", "-o",
                        os.path.join(d, "p.o")], check=True)
    lib = api.capi()
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    assert lib.blance_plan_chains_ex.argtypes == [vp, vp, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp,
                                                  vp, vp, vp]
    assert lib.blance_plan_chains_ex.argtypes == lib.blance_plan_chains_exposure.argtypes
    assert NAME in api.EXPORTS


# ---- argument errors without a device ---------------------------------------------------------------------------

class _StageCall(_Call):
    """A _Call of blance_plan_chains_ex: stage_opts [n][T], the bad options at chain 1, stage `at` (default 1)."""

    def __init__(self, stage_opts=None, at=1, **kw):
        super().__init__(True, **kw)
        m, T = max(1, self.n), max(1, self.T)
        self.stage_opts = None
        self.keep = []
        if stage_opts is not None:
            self.stage_opts = (api.ScenarioOpts * (m * T))()
            for k, v in stage_opts.items():
                if isinstance(v, (list, tuple)):
                    a = np.ascontiguousarray(v, np.uint8 if k in ("state_has_stickiness", "ow_has") else
                                             np.uint32 if k == "ie_mask" else np.int32)
                    self.keep.append(a)
                    v = a.ctypes.data
                setattr(self.stage_opts[min(1, m - 1) * T + min(at, T - 1)], k, v)


def _invoke(c):
    return api.capi().blance_plan_chains_ex(None, c.base_p, c.n, c.T, c.stages_p, c.stage_opts, 0, 0, c.nmc, c.mc, None, c.out, c.net,
                                           c.sched, ctypes.byref(c.aopts), c.audit, c.eopts_p, c.series_cap, c.expo, c.net_sched,
                                           c.net_expo, c.span)


C_ = api.OPT_CONSTRAINTS
S_ = api.OPT_STICKINESS
W_ = api.OPT_PART_WEIGHTS
H_ = api.OPT_HIERARCHY
NO_SCHED = dict(nmc=0, mc=False, sched=False, expo=False)
NEED_SCHED = (INVALID, NAME + ": expo, net_sched, net_expo and span need a schedule")


def _stage(msg, st=INVALID, chain=1, stage=1):
    return (st, "%s: chain %d, stage %d: %s" % (NAME, chain, stage, msg))


# (row name, knobs, (status, message), schedule outputs cleared); _base() has 2 states of one slot each, 6 partitions
ROWS = [
    ("ok", {}, NULL_CTX, 8),
    ("ok without stage options", dict(stage_opts=None), NULL_CTX, 8),
    ("everything", dict(net_sched=True, net_expo=True, span="dom_peak", series_cap=3), NULL_CTX, 8),
    ("no schedule", dict(NO_SCHED), NULL_CTX, 0),
    ("no schedule, an audit", dict(NO_SCHED, audit=True), NULL_CTX, 0),
    ("no schedule, expo", dict(NO_SCHED, expo=True), NEED_SCHED, 0),
    ("no schedule, net_sched", dict(NO_SCHED, net_sched=True), NEED_SCHED, 0),
    ("no schedule, span", dict(NO_SCHED, span="part_done_round"), NEED_SCHED, 0),
    ("n_move_conc without a schedule", dict(nmc=0), (INVALID, NAME + ": n_move_conc must be positive"), 0),
    ("sched without move_conc", dict(mc=False), (INVALID, NAME + ": n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("n", dict(n=0), (INVALID, NAME + ": n must be positive"), 0),
    ("n_stages", dict(T=0), (INVALID, NAME + ": n_stages must be positive"), 0),
    ("base", dict(base=False), (INVALID, NAME + ": base, stages or out is NULL"), 0),
    ("stages", dict(sc=False), (INVALID, NAME + ": base, stages or out is NULL"), 8),
    ("max_iters", dict(max_iters=0), (INVALID, NAME + ": a chain of several stages needs max_iters >= 1"), 8),
    ("stage", BAD_SCEN, _stage("add_is_nil is neither 0 nor 1"), 8),
    ("net_sched without net", dict(net=False, net_sched=True), (INVALID, NAME + ": net_sched and net_expo need net"), 0),
    ("event bound", dict(dom=True, n_parts=EVENTS_OVER, audit=False),
     (UNSUPPORTED, NAME + ": chain 1, stage 1, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31"), 8),
    ("eopts forest", dict(eopts="cycle"),
     (INVALID, NAME + ": domain_parent has a cycle or a vertex more than 16 edges below its root (vertex 0)"), 8),
    # one row per option group and bad value, at chain 1, stage 1 (stage 0 of chain 1 is valid)
    ("set", dict(stage_opts=dict(set=0x100)), _stage("opts.set has an unknown bit"), 8),
    ("constraints beyond the slot range", dict(stage_opts=dict(set=C_, state_constraints=[2, 1])),
     _stage("a state's slot range is smaller than its constraints"), 8),
    ("constraints NULL", dict(stage_opts=dict(set=C_), audit=False), _stage("state tables are NULL"), 8),
    ("stickiness flag", dict(stage_opts=dict(set=S_, state_stickiness=[1, 1], state_has_stickiness=[1, 2])),
     _stage("state_has_stickiness is neither 0 nor 1"), 8),
    ("has_part_weights", dict(stage_opts=dict(set=W_, has_part_weights=2)), _stage("has_part_weights is neither 0 nor 1"), 8),
    ("n_weight_overrides", dict(stage_opts=dict(set=W_, n_weight_overrides=-1)), _stage("n_weight_overrides is negative"), 8),
    ("override arrays", dict(stage_opts=dict(set=W_, n_weight_overrides=1)), _stage("weight override arrays are NULL"), 8),
    ("override outside", dict(stage_opts=dict(set=W_, n_weight_overrides=1, ow_part=[6], ow_weight=[1], ow_has=[1])),
     _stage("a weight override's partition is outside [0, n_parts)"), 8),
    ("override twice", dict(stage_opts=dict(set=W_, n_weight_overrides=2, ow_part=[3, 3], ow_weight=[1, 2], ow_has=[1, 1])),
     _stage("a partition has two weight overrides"), 8),
    ("ow_has", dict(stage_opts=dict(set=W_, n_weight_overrides=1, ow_part=[0], ow_weight=[1], ow_has=[2])),
     _stage("ow_has is neither 0 nor 1"), 8),
    ("weight above 999999999", dict(stage_opts=dict(set=W_, n_weight_overrides=1, ow_part=[0], ow_weight=[1000000000], ow_has=[1])),
     _stage("partition weight above 999999999 in override 0", UNSUPPORTED), 8),
    ("count bound", dict(stage_opts=dict(set=W_, has_part_weights=1, n_weight_overrides=3, ow_part=[0, 1, 2],
                                         ow_weight=[999999999] * 3, ow_has=[1] * 3)), _stage(COUNT_BOUND, UNSUPPORTED), 8),
    ("has_hier_rules", dict(stage_opts=dict(set=H_, has_hier_rules=2, n_hier_bits=4, rule_off=[0, 0, 0]), audit=False),
     _stage("has_hier_rules is neither 0 nor 1"), 8),
    ("rule_off NULL", dict(stage_opts=dict(set=H_, has_hier_rules=1), audit=False), _stage("rule_off is NULL"), 8),
    # the audit model is checked at every stage, before the schedule request
    ("audit model", dict(stage_opts=dict(set=H_, has_hier_rules=1)), _stage("rule_off is NULL"), 0),
    ("audit model at stage 0", dict(stage_opts=dict(set=H_, has_hier_rules=1), at=0), _stage("rule_off is NULL", stage=0), 0),
    ("options at stage 0", dict(stage_opts=dict(set=0x100), at=0), _stage("opts.set has an unknown bit", stage=0), 8),
    # two bad arguments: which check fires first
    ("stage before options", dict(BAD_SCEN, stage_opts=dict(set=0x100)), _stage("add_is_nil is neither 0 nor 1"), 8),
    ("schedule before options", dict(nmc=0, stage_opts=dict(set=0x100)), (INVALID, NAME + ": n_move_conc must be positive"), 0),
    ("audit flags before no schedule, expo", dict(NO_SCHED, expo=True, aflags=0x80), (INVALID, NAME + ": audit flags hold an unknown bit"), 0),
    ("audit model before no schedule, expo", dict(NO_SCHED, expo=True, stage_opts=dict(set=H_, has_hier_rules=1)), _stage("rule_off is NULL"), 0),
]


@pytest.mark.parametrize("name,knobs,want,cleared", ROWS, ids=[r[0] for r in ROWS])
def test_null_context_row(name, knobs, want, cleared):
    kw = dict(knobs)
    kw.setdefault("stage_opts", {})
    if kw.get("eopts") == "cycle":
        kw["eopts"] = _cycle()
    c = _StageCall(**kw)
    st = _invoke(c)
    assert (st, api.capi().blance_last_error(None).decode()) == want
    assert c.cleared() == cleared


def test_python_wrapper_errors():
    from blance_b200 import tables
    t = tables.PlanTables(4, 2, 6, [0, 1], [1, 1])
    ctx = tables.Context.__new__(tables.Context)
    ctx.lib, ctx.ptr, ctx._rounds = api.capi(), ctypes.c_void_p(), {}
    with pytest.raises(ValueError, match="not both"):
        ctx.plan_chains(t, [[{}]], False, opts=[{}], stage_opts=[[{}]])
    with pytest.raises(ValueError, match="one option dict per stage"):
        ctx.plan_chains(t, [[{}, {}]], False, stage_opts=[[{}]])
    with pytest.raises(blance_b200.BlanceError, match="blance_plan_chains_ex failed .*: ctx is NULL"):
        ctx.plan_chains(t, [[{}, {}]], False, stage_opts=[[{}, {}]])


# ---- the per-stage reference against the literal Go loop --------------------------------------------------------

def check_chain(kw, seed):
    if not removal_allowed(kw) and kw["nodes_to_remove"]:
        return 0
    stages = make_chain(kw, seed)
    if not removal_allowed(kw):       # plan.go:544 panics on a removal in stage 1 only
        stages[0] = (stages[0][0], [], stages[0][2], stages[0][3])
    keys = CS.make_stage_options(kw, seed, len(stages))
    lit = CS.literal_chain_staged(kw, stages, keys)
    base, chain, opts, ips = CS.staged_flat_chain(kw, stages, keys)
    ref, net = CS.chain_reference_staged(base, chain, opts, bool(seed % 2))
    for t, (l, r) in enumerate(zip(lit, ref)):
        next_map, warnings = unintern(ips[t], t, r)    # warnings name the stage's own constraints
        assert next_map == l["next_map"], (seed, t, keys)
        assert warnings == l["warnings"], (seed, t, keys)
        assert r["iters_run"] == l["iterations"], (seed, t)
    assert net["ops_total"] == int(net["node_ops"].sum())
    return sum(1 for k in keys if k)


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_staged_reference_matches_literal_loop_golden(c):
    check_chain(G.plan_kwargs(c), c["index"])


@pytest.mark.parametrize("chunk", range(4))
def test_staged_reference_matches_literal_loop_random(chunk):
    varied = 0
    for seed in range(chunk * 40, (chunk + 1) * 40):
        varied += check_chain(random_instance(seed), seed)
    assert varied > 20                 # most chains set options at some stage


def test_every_pattern_is_exercised():
    """The four per-stage patterns occur with their intended shape on the random instances."""
    seen = set()
    for seed in range(40):
        kw = random_instance(seed)
        keys = CS.make_stage_options(kw, seed, 3)
        if "modelStateConstraints" in keys[1] and not keys[2]:
            seen.add("constraints up at stage 1, back at stage 2")
        if any("stateStickiness" in k for k in keys):
            seen.add("stickiness at one stage")
        if "partitionWeights" in keys[0] and keys[2].get("partitionWeights", 0) is None:
            seen.add("weights at stage 0, back at 1, nil at 2")
        if keys[0].get("hierarchyRules", 0) is None and keys[2].get("hierarchyRules"):
            seen.add("rules first at the last stage")
    assert len(seen) == 4, seen


def test_string_face_rejects_stage_options_before_device_work():
    prev = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}}
    model = {"primary": (0, 1)}
    stages = [{"nodesToRemove": [], "nodesToAdd": None},
              {"nodesToRemove": [], "nodesToAdd": None, "modelStateConstraints": {"primary": 17}}]
    with pytest.raises(blance_b200.BlanceError, match="constraints 17"):
        blance_b200.PlanNextMapChains(prev, prev, ["a", "b"], model, None, [{"stages": stages}])
    stages[1] = {"nodesToRemove": [], "nodesToAdd": None, "partitionWeights": {"1": 1000000000}}
    with pytest.raises(blance_b200.BlanceError, match="chain 0, stage 1: partition weight of '1'"):
        blance_b200.PlanNextMapChains(prev, prev, ["a", "b"], model, None, [{"stages": stages}])
