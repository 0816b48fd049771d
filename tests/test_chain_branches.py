"""What-if branches off the stages of a chain (blance_plan_chain_branches), CPU side: the ctypes declaration against the
header, and every argument error with a NULL context, one row per bad argument, each branch-stage error naming the
branch and its stage.  The device path is tests/test_chain_branches_gpu.py."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_chain_options import _StageCall
from test_wave_requests import INVALID, NULL_CTX, UNSUPPORTED

from blance_b200 import abi as api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "blance_plan_chain_branches"


def test_declaration_matches_header():
    decl = r'''
    #include "blance_b200.h"
    typedef int (*fn)(blance_ctx*, const blance_plan_in*, int32_t, int32_t, const blance_chain_stage*, const blance_scenario_opts*,
                      int32_t, int32_t, int32_t, const int32_t*, const uint8_t*, blance_scenario_out*, blance_chain_out*,
                      blance_scenario_schedule_out*, const blance_audit_opts*, blance_audit_out*, const blance_audit_opts*,
                      int32_t, blance_exposure_out*, blance_scenario_schedule_out*, blance_exposure_out*, blance_chain_span_out*,
                      int32_t, int32_t, const blance_chain_branch*, blance_scenario_out*, blance_chain_out*,
                      blance_scenario_schedule_out*, blance_audit_out*, blance_exposure_out*, blance_scenario_schedule_out*,
                      blance_exposure_out*);
    int main(void) { fn f = blance_plan_chain_branches; (void)f; return 0; }
    '''
    layout = r'''
    #include <stddef.h>
    #include <stdio.h>
    #include "blance_b200.h"
    int main(void) {
      printf("%zu %zu %zu %zu\n", sizeof(blance_chain_branch), offsetof(blance_chain_branch, after_stage),
             offsetof(blance_chain_branch, stages), offsetof(blance_chain_branch, stage_opts));
      return 0;
    }
    '''
    inc = ["-I", os.path.join(ROOT, "include")]
    with tempfile.TemporaryDirectory() as d:
        c, e = os.path.join(d, "p.c"), os.path.join(d, "e.c")
        open(c, "w").write(decl)
        open(e, "w").write(layout)
        # -Werror: a prototype that differs from the typedef in any argument does not compile
        subprocess.run(["gcc", "-Werror", "-Wincompatible-pointer-types"] + inc + [c, "-c", "-o", os.path.join(d, "p.o")], check=True)
        subprocess.run(["gcc"] + inc + [e, "-o", os.path.join(d, "e")], check=True)
        sizes = [int(x) for x in subprocess.run([os.path.join(d, "e")], check=True, capture_output=True, text=True).stdout.split()]
    B = api.ChainBranch
    assert sizes == [ctypes.sizeof(B), B.after_stage.offset, B.stages.offset, B.stage_opts.offset]
    lib = api.capi()
    i32, vp = ctypes.c_int32, ctypes.c_void_p
    assert lib.blance_plan_chain_branches.argtypes == lib.blance_plan_chains_ex.argtypes + [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    assert NAME in api.EXPORTS


class _BranchCall(_StageCall):
    """A _StageCall of the trunk plus nb branches of TB stages each; branch 1, stage `bat` carries the bad branch
    scenario or options."""

    def __init__(self, nb=2, TB=1, chain=0, after=0, br=True, br_out=True, bstages=True, bscen=None, bopts=None, bat=0,
                 br_net=True, br_sched=None, br_audit=False, br_expo=False, br_net_sched=False, br_net_expo=False, **kw):
        super().__init__(**kw)
        b = self.base
        m, mt = max(1, nb), max(1, TB)
        self.nb, self.TB = nb, TB
        self.bst = (api.ChainStage * (m * mt))()
        for x in range(m * mt):
            s = self.bst[x]
            s.nodes.node_removed, s.nodes.node_added = b.node_removed, b.node_added
            s.node_in_all = self.in_all.ctypes.data
        for k, v in (bscen or {}).items():
            setattr(self.bst[min(1, m - 1) * mt + bat].nodes, k, v)
        self.bopts = (api.ScenarioOpts * (m * mt))()
        for k, v in (bopts or {}).items():
            if isinstance(v, (list, tuple)):
                a = np.ascontiguousarray(v, np.uint8 if k in ("state_has_stickiness", "ow_has") else np.int32)
                self.keep.append(a)
                v = a.ctypes.data
            setattr(self.bopts[min(1, m - 1) * mt + bat], k, v)
        self.br = (api.ChainBranch * m)()
        for x in range(m):
            self.br[x].chain, self.br[x].after_stage = chain if x == 1 else 0, after if x == 1 else 0
            self.br[x].stages = ctypes.addressof(self.bst[x * mt]) if bstages else None
            self.br[x].stage_opts = ctypes.addressof(self.bopts[x * mt])
        nc = max(1, min(self.nmc, 8))
        if br_sched is None:
            br_sched = self.sched is not None
        self.br_p = self.br if br else None
        self.br_out = (api.ScenarioOut * (m * mt))() if br_out else None
        self.br_net = (api.ChainOut * m)() if br_net else None
        self.br_sched = (api.ScenarioScheduleOut * (m * mt * nc))() if br_sched else None
        self.br_audit = (api.AuditOut * (m * mt))() if br_audit else None
        self.br_expo = (api.ExposureOut * (m * mt * nc))() if br_expo else None
        self.br_net_sched = (api.ScenarioScheduleOut * (m * nc))() if br_net_sched else None
        self.br_net_expo = (api.ExposureOut * (m * nc))() if br_net_expo else None


def _invoke(c):
    return api.capi().blance_plan_chain_branches(
        None, c.base_p, c.n, c.T, c.stages_p, c.stage_opts, 0, 0, c.nmc, c.mc, None, c.out, c.net, c.sched, ctypes.byref(c.aopts),
        c.audit, c.eopts_p, c.series_cap, c.expo, c.net_sched, c.net_expo, c.span, c.nb, c.TB, c.br_p, c.br_out, c.br_net, c.br_sched,
        c.br_audit, c.br_expo, c.br_net_sched, c.br_net_expo)


NO_SCHED = dict(nmc=0, mc=False, sched=False, expo=False)
NEED_SCHED = (INVALID, NAME + ": br_sched, br_expo, br_net_sched and br_net_expo need a schedule")
NEED_EXPO = (INVALID, NAME + ": br_expo needs expo and br_net_expo needs br_expo")


def _at(msg, st=INVALID, branch=1, stage=0):
    return (st, "%s: branch %d, stage %d: %s" % (NAME, branch, stage, msg))


def _br(msg, branch=1):
    return (INVALID, "%s: branch %d: %s" % (NAME, branch, msg))


# (row name, knobs, (status, message)); the trunk is test_chain_options' valid call: 2 chains of 2 stages, 6 partitions
ROWS = [
    ("ok", {}, NULL_CTX),
    ("no branches", dict(nb=0, br=False, br_out=False, br_sched=False), NULL_CTX),
    ("everything", dict(TB=2, after=1, chain=1, br_audit=True, br_expo=True, br_net_sched=True, br_net_expo=True, net_expo=True,
                        series_cap=3), NULL_CTX),
    ("from the base", dict(after=-1), NULL_CTX),
    ("no schedule", dict(NO_SCHED), NULL_CTX),
    ("no schedule, br_audit", dict(NO_SCHED, br_audit=True), NULL_CTX),
    # the trunk's checks come first
    ("trunk stage before branches", dict(nb=-1, scen=dict(add_is_nil=2)),
     (INVALID, "blance_plan_chain_branches: chain 1, stage 1: add_is_nil is neither 0 nor 1")),
    ("n_branches", dict(nb=-1), (INVALID, NAME + ": n_branches is negative")),
    ("n_branch_stages", dict(TB=0), (INVALID, NAME + ": n_branch_stages must be positive")),
    ("br", dict(br=False), (INVALID, NAME + ": br or br_out is NULL")),
    ("br_out", dict(br_out=False), (INVALID, NAME + ": br or br_out is NULL")),
    ("br_net_sched without br_net", dict(br_net=False, br_net_sched=True), (INVALID, NAME + ": br_net_sched and br_net_expo need br_net")),
    ("br_net_expo without br_net", dict(br_net=False, br_net_expo=True, br_expo=True),
     (INVALID, NAME + ": br_net_sched and br_net_expo need br_net")),
    ("br_sched missing", dict(br_sched=False), (INVALID, NAME + ": br_sched is NULL with a schedule")),
    ("br_sched without a schedule", dict(NO_SCHED, br_sched=True), NEED_SCHED),
    ("br_expo without a schedule", dict(NO_SCHED, br_expo=True), NEED_SCHED),
    ("br_net_sched without a schedule", dict(NO_SCHED, br_net_sched=True), NEED_SCHED),
    ("br_expo without expo", dict(expo=False, br_expo=True), NEED_EXPO),
    ("br_net_expo without br_expo", dict(br_net_expo=True), NEED_EXPO),
    ("stages", dict(bstages=False), _br("stages is NULL", branch=0)),
    ("chain below 0", dict(chain=-1), _br("chain outside [0, n)")),
    ("chain at n", dict(chain=2), _br("chain outside [0, n)")),
    ("after_stage below -1", dict(after=-2), _br("after_stage outside [-1, n_stages)")),
    ("after_stage at n_stages", dict(after=2), _br("after_stage outside [-1, n_stages)")),
    ("max_iters", dict(max_iters=0, T=1, after=0), _br("a chain of several stages needs max_iters >= 1", branch=0)),
    ("branch stage", dict(bscen=dict(add_is_nil=2)), _at("add_is_nil is neither 0 nor 1")),
    ("branch stage 1", dict(TB=2, bscen=dict(add_is_nil=2), bat=1), _at("add_is_nil is neither 0 nor 1", stage=1)),
    ("node weights flag", dict(bscen=dict(has_node_weights=3)), _at("has_node_weights is neither 0 nor 1")),
    ("branch options", dict(bopts=dict(set=0x100)), _at("opts.set has an unknown bit")),
    ("branch constraints", dict(TB=2, bat=1, bopts=dict(set=api.OPT_CONSTRAINTS, state_constraints=[2, 1])),
     _at("a state's slot range is smaller than its constraints", stage=1)),
    ("branch weight", dict(bopts=dict(set=api.OPT_PART_WEIGHTS, n_weight_overrides=1, ow_part=[0], ow_weight=[1000000000], ow_has=[1])),
     _at("partition weight above 999999999 in override 0", UNSUPPORTED)),
    ("branch audit model", dict(br_audit=True, bopts=dict(set=api.OPT_HIERARCHY, has_hier_rules=1, n_hier_bits=4)),
     _at("rule_off is NULL")),
    ("branch event bound", dict(br_expo=True, br_dom=True),
     (UNSUPPORTED, NAME + ": branch 1, stage 0, count 1: dom_peak needs 2 x 17 x 2 x n_slots x n_parts < 2^31")),
    # without a trunk audit, the audit options are first checked for br_audit
    ("branch audit flags", dict(audit=False, aflags=0x80, br_audit=True), (INVALID, NAME + ": audit flags hold an unknown bit")),
    # two bad arguments: which check fires first
    ("chain before branch stage", dict(chain=-1, bscen=dict(add_is_nil=2)), _br("chain outside [0, n)")),
    ("branch stage before audit flags", dict(audit=False, aflags=0x80, br_audit=True, bscen=dict(add_is_nil=2)),
     _at("add_is_nil is neither 0 nor 1")),
    ("branch audit model before branch event bound",
     dict(br_audit=True, br_expo=True, br_dom=True, bopts=dict(set=api.OPT_HIERARCHY, has_hier_rules=1, n_hier_bits=4)),
     _at("rule_off is NULL")),
]


@pytest.mark.parametrize("name,knobs,want", ROWS, ids=[r[0] for r in ROWS])
def test_null_context_row(name, knobs, want):
    kw = dict(knobs)
    kw.setdefault("stage_opts", {})
    br_dom = kw.pop("br_dom", False)
    c = _BranchCall(**kw)
    if br_dom:                         # 2 slots: the event bound of 2 x 17 x 2 x n_slots x n_parts
        c.base.n_parts = (1 << 31) // 136 + 1
        c.br_expo[len(c.br_expo) - 1].dom_peak = c.buf.ctypes.data
    st = _invoke(c)
    assert (st, api.capi().blance_last_error(None).decode()) == want


def test_branch_schedule_outputs_are_cleared():
    c = _BranchCall(TB=2)
    for s in c.br_sched:
        s.rounds = 99
    assert _invoke(c) == INVALID
    assert all(s.rounds == 0 for s in c.br_sched)


# ---- the string face: branch errors before any device work ------------------------------------------------------

def _string_call(branches):
    import blance_b200
    prev = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}}
    stage = {"nodesToRemove": [], "nodesToAdd": None}
    return blance_b200.PlanNextMapChains(prev, prev, ["a", "b", "c"], {"primary": (0, 1)}, None, [{"stages": [stage, stage]}],
                                         branches=branches)


@pytest.mark.parametrize("branches,msg", [
    ([{"chain": 1, "afterStage": 0, "stages": [{"nodesToRemove": [], "nodesToAdd": None}]}], "branch 0: Chain outside"),
    ([{"chain": 0, "afterStage": 2, "stages": [{"nodesToRemove": [], "nodesToAdd": None}]}], "branch 0: AfterStage outside"),
    ([{"chain": 0, "afterStage": -2, "stages": [{"nodesToRemove": [], "nodesToAdd": None}]}], "branch 0: AfterStage outside"),
    ([{"chain": 0, "afterStage": 0, "stages": []}], "branch 0 has 0 stages"),
    ([{"chain": 0, "afterStage": 0, "stages": [{"nodesToRemove": [], "nodesToAdd": None}]},
      {"chain": 0, "afterStage": 1, "stages": [{"nodesToRemove": [], "nodesToAdd": None}] * 2}], "branch 1 has 2 stages"),
    ([{"chain": 0, "afterStage": 0, "stages": [{"nodesToRemove": [], "nodesToAdd": None, "nodesAll": ["a", "z"]}]}],
     "branch 0, stage 0: NodesAll name 'z' is not in nodesAll"),
    ([{"chain": 0, "afterStage": -1, "stages": [{"nodesToRemove": [], "nodesToAdd": None},
                                                 {"nodesToRemove": [], "nodesToAdd": None,
                                                  "modelStateConstraints": {"primary": 17}}]}], "constraints 17"),
])
def test_string_face_rejects_branches_before_device_work(branches, msg):
    import blance_b200
    with pytest.raises(blance_b200.BlanceError, match=msg):
        _string_call(branches)


def test_string_face_branch_stage_needs_node_sets():
    with pytest.raises(ValueError, match="branch 0, stage 0 lacks nodesToAdd"):
        _string_call([{"chain": 0, "afterStage": 0, "stages": [{"nodesToRemove": []}]}])
