"""Flat planner tables in numpy, laid out exactly as struct blance_plan_in /
blance_plan_out of include/blance_b200.h, for callers that already hold ids
instead of strings (bench.py, the large parity tests).  The arrays are plain host
memory; PlanTables.struct() returns the ctypes struct whose pointers alias them."""
import copy
import ctypes

import numpy as np

from . import abi as api      # ctypes structs + lazy library handle: importing tables loads no native code

NO_NODE = -1
SHAPE_ABSENT, SHAPE_NIL, SHAPE_LIST = 0, 1, 2

_I32 = ("state_priority", "state_constraints", "state_slot_off", "state_stickiness", "node_weight", "part_weight",
        "part_name_rank", "prev_rows", "cur_rows", "extra_tot_first", "extra_tot_rest", "rule_off")
_U8 = ("state_has_stickiness", "node_removed", "node_added", "node_has_weight", "part_in_prev", "part_in_assign",
       "part_has_weight", "prev_shape", "cur_shape")


class PlanTables:
    """Holds every array of a blance_plan_in.  Scalars are attributes; arrays are
    C-contiguous numpy arrays of the ABI's dtypes."""

    def __init__(self, n_nodes, n_states, n_parts, state_priority, state_constraints, n_node_ids=None):
        self.n_nodes = int(n_nodes)
        self.n_node_ids = int(n_node_ids if n_node_ids is not None else n_nodes)
        self.n_states = int(n_states)
        self.n_parts = int(n_parts)
        self.max_iters = 10
        self.booster_kind = 0
        self.add_is_nil = 0
        self.has_part_weights = 0
        self.has_node_weights = 0
        self.has_hier_rules = 0
        self.engine = 0
        self.n_rules = 0
        self.n_hier_bits = self.n_nodes
        S, P, N, NU = self.n_states, self.n_parts, self.n_nodes, self.n_node_ids
        self.state_priority = np.asarray(state_priority, np.int32)
        self.state_constraints = np.asarray(state_constraints, np.int32)
        caps = np.maximum(self.state_constraints, 0)
        self.state_slot_off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
        self.n_slots = int(self.state_slot_off[-1])
        self.top_state = int(np.argmin(self.state_priority)) if S else 0
        self.state_stickiness = np.zeros(S, np.int32)
        self.state_has_stickiness = np.zeros(S, np.uint8)
        self.node_removed = np.zeros(NU, np.uint8)
        self.node_added = np.zeros(NU, np.uint8)
        self.node_weight = np.zeros(N, np.int32)
        self.node_has_weight = np.zeros(N, np.uint8)
        self.part_in_prev = np.zeros(P, np.uint8)
        self.part_in_assign = np.ones(P, np.uint8)
        self.part_weight = np.ones(P, np.int32)
        self.part_has_weight = np.zeros(P, np.uint8)
        self.part_name_rank = np.arange(P, dtype=np.int32)
        self.prev_rows = np.full((P, self.n_slots), NO_NODE, np.int32)
        self.cur_rows = np.full((P, self.n_slots), NO_NODE, np.int32)
        self.prev_shape = np.zeros((P, S), np.uint8)
        self.cur_shape = np.zeros((P, S), np.uint8)
        self.extra_tot_first = np.zeros(N, np.int32)
        self.extra_tot_rest = np.zeros(N, np.int32)
        self.rule_off = np.zeros(S + 1, np.int32)
        self.ie_mask = np.zeros(0, np.uint32)

    @property
    def hier_words(self):
        return (self.n_hier_bits + 31) // 32

    def struct(self):
        s = api.PlanIn()
        for f in api._I32_FIELDS:
            setattr(s, f, int(getattr(self, f)))
        s.n_rules, s.n_hier_bits, s.engine = int(self.n_rules), int(self.n_hier_bits), int(self.engine)
        self._keep = []
        for f in api._PTR_FIELDS + ("rule_off", "ie_mask"):
            want = np.uint32 if f == "ie_mask" else (np.int32 if f in _I32 else np.uint8)
            a = np.ascontiguousarray(getattr(self, f), dtype=want)
            setattr(self, f, a)
            self._keep.append(a)
            setattr(s, f, a.ctypes.data if a.size else None)
        return s


class PlanResult:
    """Output buffers of a blance_plan_out."""

    def __init__(self, t):
        self.next_rows = np.full((t.n_parts, t.n_slots), NO_NODE, np.int32)
        self.next_shape = np.zeros((t.n_parts, t.n_states), np.uint8)
        self.warn = np.zeros((t.n_parts, t.n_states), np.uint8)
        # one spare element so zero-sized cases still have valid pointers
        self._pad = np.zeros(4, np.int32)
        self.out = api.PlanOut()
        self.out.next_rows = self.next_rows.ctypes.data if self.next_rows.size else self._pad.ctypes.data
        self.out.next_shape = self.next_shape.ctypes.data if self.next_shape.size else self._pad.ctypes.data
        self.out.warn = self.warn.ctypes.data if self.warn.size else self._pad.ctypes.data

    iters_run = property(lambda self: self.out.iters_run)
    converged = property(lambda self: self.out.converged)
    steps = property(lambda self: self.out.steps)
    sticky_steps = property(lambda self: self.out.sticky_steps)
    device_ms = property(lambda self: self.out.device_ms)
    kernel_ms = property(lambda self: self.out.kernel_ms)
    pass_ms = property(lambda self: self.out.pass_ms)


SCENARIO_FIELDS = ("node_removed", "node_added", "add_is_nil", "has_node_weights", "node_weight", "node_has_weight")


class ScenarioResult:
    """Output buffers of a blance_scenario_out: the summaries always, the next map's tables when requested."""

    def __init__(self, t, want_rows):
        self.node_ops = np.zeros((t.n_node_ids, 4), np.int64)
        self.state_node_load = np.zeros((t.n_states, t.n_node_ids), np.int64)
        self.next_rows = np.full((t.n_parts, t.n_slots), NO_NODE, np.int32) if want_rows else None
        self.next_shape = np.zeros((t.n_parts, t.n_states), np.uint8) if want_rows else None
        self.warn = np.zeros((t.n_parts, t.n_states), np.uint8) if want_rows else None
        self.out = api.ScenarioOut()
        for f in ("node_ops", "state_node_load", "next_rows", "next_shape", "warn"):
            a = getattr(self, f)
            setattr(self.out, f, a.ctypes.data if a is not None and a.size else None)

    iters_run = property(lambda self: self.out.iters_run)
    converged = property(lambda self: self.out.converged)
    steps = property(lambda self: self.out.steps)
    sticky_steps = property(lambda self: self.out.sticky_steps)
    schedules = None          # blance_plan_scenarios_schedule: one ScenarioSchedule per count
    audit = None              # blance_plan_scenarios_audit: the AuditResult of the final map
    parts_moved = property(lambda self: self.out.parts_moved)
    ops_total = property(lambda self: self.out.ops_total)
    warn_parts = property(lambda self: self.out.warn_parts)


class ChainNet:
    """Output buffers of a blance_chain_out: the moves from a chain's base map to its last stage's map."""

    def __init__(self, t):
        self.node_ops = np.zeros((t.n_node_ids, 4), np.int64)
        self.out = api.ChainOut()
        self.out.node_ops = self.node_ops.ctypes.data if self.node_ops.size else None

    ops_total = property(lambda self: self.out.ops_total)
    parts_moved = property(lambda self: self.out.parts_moved)


class ScenarioSchedule:
    """Output buffers of a blance_scenario_schedule_out: the schedule's summaries at one count."""

    def __init__(self, t, count):
        self.count = count
        self.node_rounds = np.zeros(t.n_node_ids, np.int32)
        self.node_last_round = np.zeros(t.n_node_ids, np.int32)
        self.part_done_round = np.zeros(t.n_parts, np.int32)
        self.out = api.ScenarioScheduleOut()
        for f in ("node_rounds", "node_last_round", "part_done_round"):
            a = getattr(self, f)
            setattr(self.out, f, a.ctypes.data if a.size else None)

    rounds = property(lambda self: self.out.rounds)
    moves_done = property(lambda self: self.out.moves_done)
    stuck_parts = property(lambda self: self.out.stuck_parts)
    max_batch = property(lambda self: self.out.max_batch)


class AuditResult:
    """Output buffers of a blance_audit_out for a map of `t`'s sizes with n_rules rules: every array, the failover
    matrix only with n2n."""

    def __init__(self, t, n_rules, n_domains=0, n2n=False):
        V = t.n_node_ids + n_domains
        self.short_slots = np.zeros(t.n_states, np.int64)
        self.over_slots = np.zeros(t.n_states, np.int64)
        self.rule_miss = np.zeros(n_rules, np.int64)
        self.rule_tested = np.zeros(n_rules, np.int64)
        self.dom_top = np.zeros(V, np.int64)
        self.dom_all = np.zeros(V, np.int64)
        self.dom_copies = np.zeros(V, np.int64)
        self.n2n = np.zeros((t.n_nodes, t.n_nodes), np.int32) if n2n else None
        self.part_flags = np.zeros(t.n_parts, np.uint8)
        self.out = api.AuditOut()
        for f in ("short_slots", "over_slots", "rule_miss", "rule_tested", "dom_top", "dom_all", "dom_copies", "n2n", "part_flags"):
            a = getattr(self, f)
            setattr(self.out, f, a.ctypes.data if a is not None and a.size else None)

    short_parts = property(lambda self: self.out.short_parts)
    rule_miss_parts = property(lambda self: self.out.rule_miss_parts)
    no_top_parts = property(lambda self: self.out.no_top_parts)
    n2n_max = property(lambda self: (self.out.n2n_max, self.out.n2n_max_a, self.out.n2n_max_b))
    kernel_ms = property(lambda self: self.out.kernel_ms)


def _audit_opts(n2n, domain_parent, n_node_ids, keep):
    """blance_audit_opts of (n2n, domain_parent [n_node_ids + n_domains] or None) and its n_domains."""
    o = api.AuditOpts()
    o.flags = api.AUDIT_N2N if n2n else 0
    if domain_parent is not None:
        a = np.ascontiguousarray(domain_parent, np.int32)
        keep.append(a)
        o.n_domains = a.size - n_node_ids
        o.domain_parent = a.ctypes.data
    return o, int(o.n_domains)


def _n_rules(t):
    return int(t.n_rules) if t.has_hier_rules else 0


def scenario_tables(base, scenario, opts=None):
    """The PlanTables of one scenario: `base` with the scenario's node fields substituted and, when `opts` (a dict
    of OPT_GROUPS keys) is given, its plan options: the PlanNextMapEx instance blance_plan_scenarios_ex plans.  A
    field missing from the dicts keeps the base's value.  A shallow copy: the row tables are shared with `base`,
    the weight arrays are copied when the scenario has weight overrides."""
    t = copy.copy(base)
    for f in SCENARIO_FIELDS:
        if f in scenario:
            setattr(t, f, scenario[f])
    for f, v in (opts or {}).items():
        if f not in _OPT_KEYS:
            raise KeyError("unknown scenario option %r" % f)
        if f == "weight_overrides":
            part, weight, has = (np.asarray(a) for a in v)
            t.part_weight = np.array(base.part_weight, np.int32)
            t.part_has_weight = np.array(base.part_has_weight, np.uint8)
            t.part_weight[part] = weight
            t.part_has_weight[part] = has
        elif v is not None:                  # (extra_tot_* None: the base's)
            setattr(t, f, v)
    return t


def widen_layout(t, widths):
    """A copy of `t` whose state s has a slot range of at least widths[s] (the row tables re-laid out, padded with
    NO_NODE): the shared layout of scenarios that raise a state's constraints."""
    caps = np.maximum(np.diff(t.state_slot_off), np.asarray(widths, np.int64)).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(caps)]).astype(np.int32)
    w = copy.copy(t)
    w.state_slot_off, w.n_slots = off, int(off[-1])
    for f in ("prev_rows", "cur_rows"):
        old = np.asarray(getattr(t, f)).reshape(t.n_parts, t.n_slots)
        new = np.full((t.n_parts, w.n_slots), NO_NODE, np.int32)
        for s in range(t.n_states):
            lo, hi = int(t.state_slot_off[s]), int(t.state_slot_off[s + 1])
            new[:, off[s]:off[s] + hi - lo] = old[:, lo:hi]
        setattr(w, f, new)
    return w


# blance_scenario_opts in dict form: the keys of each group (a group is set when any of its keys is given)
OPT_GROUPS = {api.OPT_CONSTRAINTS: ("state_constraints",),
              api.OPT_STICKINESS: ("state_stickiness", "state_has_stickiness"),
              api.OPT_PART_WEIGHTS: ("has_part_weights", "weight_overrides", "extra_tot_first", "extra_tot_rest"),
              api.OPT_HIERARCHY: ("has_hier_rules", "n_rules", "n_hier_bits", "rule_off", "ie_mask")}
_OPT_KEYS = {k for keys in OPT_GROUPS.values() for k in keys}


def _opts_struct(base, o, keep):
    """blance_scenario_opts of one option dict (weight_overrides = (partitions, weights, presence))."""
    s = api.ScenarioOpts()
    for bit, keys in OPT_GROUPS.items():
        if any(k in o for k in keys):
            s.set |= bit

    def ptr(v, dt):
        a = np.ascontiguousarray(v, dtype=dt)
        keep.append(a)
        return a.ctypes.data if a.size else None
    if s.set & api.OPT_CONSTRAINTS:
        s.state_constraints = ptr(o["state_constraints"], np.int32)
    if s.set & api.OPT_STICKINESS:
        s.state_stickiness = ptr(o.get("state_stickiness", base.state_stickiness), np.int32)
        s.state_has_stickiness = ptr(o.get("state_has_stickiness", base.state_has_stickiness), np.uint8)
    if s.set & api.OPT_PART_WEIGHTS:
        s.has_part_weights = int(o.get("has_part_weights", base.has_part_weights))
        part, weight, has = o.get("weight_overrides", ((), (), ()))
        s.n_weight_overrides = len(part)
        s.ow_part, s.ow_weight, s.ow_has = ptr(part, np.int32), ptr(weight, np.int32), ptr(has, np.uint8)
        for f in ("extra_tot_first", "extra_tot_rest"):
            if o.get(f) is not None:
                setattr(s, f, ptr(o[f], np.int32))
    if s.set & api.OPT_HIERARCHY:
        s.has_hier_rules = int(o.get("has_hier_rules", base.has_hier_rules))
        s.n_rules = int(o.get("n_rules", base.n_rules))
        s.n_hier_bits = int(o.get("n_hier_bits", base.n_hier_bits))
        s.rule_off = ptr(o.get("rule_off", base.rule_off), np.int32)
        s.ie_mask = ptr(o.get("ie_mask", base.ie_mask), np.uint32)
    return s


class Context:
    """A blance_ctx* (one per process/GPU)."""

    def __init__(self, device_id=-1, device_ids=None):
        """device_ids (a list) creates a multi-GPU context: batches are sharded over those devices."""
        self.lib = api.capi()
        self.ptr = ctypes.c_void_p()
        self._rounds = {}                     # moves handle -> R of its last moves_schedule
        if device_ids is not None:
            arr = (ctypes.c_int * len(device_ids))(*device_ids)
            st = self.lib.blance_ctx_create_multi(ctypes.byref(self.ptr), arr, len(device_ids))
        else:
            st = self.lib.blance_ctx_create(ctypes.byref(self.ptr), device_id)
        if st != 0:
            raise api.BlanceError("blance_ctx_create failed (%d): %s" % (st, self.lib.blance_last_error(None).decode()))

    def device_count(self):
        return int(self.lib.blance_ctx_device_count(self.ptr))

    def _check(self, st, what):
        if st != 0:
            raise api.BlanceError("%s failed (%d): %s" % (what, st, self.lib.blance_last_error(self.ptr).decode()))

    def plan_next_map(self, tables, result=None):
        """blance_plan_next_map: host buffers in, host buffers out."""
        result = result or PlanResult(tables)
        s = tables.struct()
        self._check(self.lib.blance_plan_next_map(self.ptr, ctypes.byref(s), ctypes.byref(result.out)), "blance_plan_next_map")
        return result

    def plan_next_map_batch(self, tables_list, results=None):
        n = len(tables_list)
        results = results or [PlanResult(t) for t in tables_list]
        ins = (api.PlanIn * n)(*[t.struct() for t in tables_list])
        outs = (api.PlanOut * n)(*[r.out for r in results])
        self._check(self.lib.blance_plan_next_map_batch(self.ptr, n, ins, outs), "blance_plan_next_map_batch")
        for r, o in zip(results, outs):
            r.out = o
        return results

    def map_audit(self, tables, rows, shape, n2n=False, domain_parent=None):
        """blance_map_audit of the map (rows [n_parts][n_slots], shape [n_parts][n_states]) against the model and
        hierarchy of `tables`.  Returns an AuditResult."""
        keep = []
        o, n_dom = _audit_opts(n2n, domain_parent, tables.n_node_ids, keep)
        r = AuditResult(tables, _n_rules(tables), n_dom, n2n)
        rows = np.ascontiguousarray(rows, np.int32)
        shape = np.ascontiguousarray(shape, np.uint8)
        s = tables.struct()
        self._check(self.lib.blance_map_audit(self.ptr, ctypes.byref(s), rows.ctypes.data if rows.size else None,
                                              shape.ctypes.data if shape.size else None, ctypes.byref(o), ctypes.byref(r.out)),
                    "blance_map_audit")
        return r

    def plan_audit(self, plan, tables, n2n=False, domain_parent=None):
        """blance_plan_audit of the resident plan `plan` (uploaded from `tables`)."""
        keep = []
        o, n_dom = _audit_opts(n2n, domain_parent, tables.n_node_ids, keep)
        r = AuditResult(tables, _n_rules(tables), n_dom, n2n)
        self._check(self.lib.blance_plan_audit(self.ptr, plan, ctypes.byref(o), ctypes.byref(r.out)), "blance_plan_audit")
        return r

    def plan_scenarios(self, base_tables, scenarios, favor_min_nodes, max_concurrent=0, want_rows=(), opts=None,
                       schedule=None, node_has_mover=None, audit=None):
        """blance_plan_scenarios: what-if variants of one cluster.  A scenario is a dict of SCENARIO_FIELDS
        (missing keys keep the base's value); want_rows lists the scenarios whose next rows, shapes and warnings
        are copied out.  opts (None, or one dict of OPT_GROUPS keys per scenario) calls blance_plan_scenarios_ex
        with those plan options.  schedule (None, or a list of MaxConcurrentPartitionMovesPerNode values) calls
        blance_plan_scenarios_schedule instead, with node_has_mover ([n_node_ids], None = the ids < n_nodes), and
        sets each result's `schedules` to one ScenarioSchedule per value.  Returns one ScenarioResult per
        scenario.  audit (None, or a dict with the optional keys n2n and domain_parent) calls
        blance_plan_scenarios_audit (with the schedules when `schedule` is given) and sets each result's `audit` to
        the AuditResult of that scenario's final map."""
        n = len(scenarios)
        want = set(want_rows)
        base = base_tables.struct()
        keep, scs = [], (api.Scenario * max(1, n))()
        for i, sc in enumerate(scenarios):
            t = scenario_tables(base_tables, sc)
            for f in SCENARIO_FIELDS:
                v = getattr(t, f)
                if f in ("add_is_nil", "has_node_weights"):
                    setattr(scs[i], f, int(v))
                    continue
                a = np.ascontiguousarray(v, dtype=np.int32 if f == "node_weight" else np.uint8)
                keep.append(a)
                setattr(scs[i], f, a.ctypes.data if a.size else None)
        results = [ScenarioResult(base_tables, i in want) for i in range(n)]
        outs = (api.ScenarioOut * max(1, n))(*[r.out for r in results])
        if schedule is not None or audit is not None:
            counts = np.ascontiguousarray([] if schedule is None else schedule, np.int32)
            mover = None if node_has_mover is None else np.ascontiguousarray(node_has_mover, np.uint8)
            if mover is not None and mover.size != base_tables.n_node_ids:
                raise ValueError("node_has_mover must have n_node_ids = %d entries" % base_tables.n_node_ids)
            sch = None
            if schedule is not None:
                for r in results:
                    r.schedules = [ScenarioSchedule(base_tables, int(c)) for c in counts]
                sch = (api.ScenarioScheduleOut * max(1, n * counts.size))(*[s.out for r in results for s in r.schedules])
            ops = None if opts is None else (api.ScenarioOpts * max(1, n))(*[_opts_struct(base_tables, o, keep) for o in opts])
            args = (self.ptr, ctypes.byref(base), n, scs, ops, int(bool(favor_min_nodes)), int(max_concurrent), int(counts.size),
                    counts.ctypes.data if counts.size else None, None if mover is None else mover.ctypes.data, outs, sch)
            if audit is None:
                self._check(self.lib.blance_plan_scenarios_schedule(*args), "blance_plan_scenarios_schedule")
            else:
                a_opts, n_dom = _audit_opts(audit.get("n2n", False), audit.get("domain_parent"), base_tables.n_node_ids, keep)
                for i, r in enumerate(results):
                    t = scenario_tables(base_tables, scenarios[i], None if opts is None else opts[i])
                    r.audit = AuditResult(base_tables, _n_rules(t), n_dom, audit.get("n2n", False))
                auds = (api.AuditOut * max(1, n))(*[r.audit.out for r in results])
                self._check(self.lib.blance_plan_scenarios_audit(*args, ctypes.byref(a_opts), auds), "blance_plan_scenarios_audit")
                for r, a in zip(results, auds):
                    r.audit.out = a
            for i, r in enumerate(results):
                for k, s in enumerate(r.schedules or ()):
                    s.out = sch[i * counts.size + k]
        elif opts is None:
            self._check(self.lib.blance_plan_scenarios(self.ptr, ctypes.byref(base), n, scs, int(bool(favor_min_nodes)),
                                                       int(max_concurrent), outs), "blance_plan_scenarios")
        else:
            ops = (api.ScenarioOpts * max(1, n))(*[_opts_struct(base_tables, o, keep) for o in opts])
            self._check(self.lib.blance_plan_scenarios_ex(self.ptr, ctypes.byref(base), n, scs, ops, int(bool(favor_min_nodes)),
                                                          int(max_concurrent), outs), "blance_plan_scenarios_ex")
        for r, o in zip(results, outs):
            r.out = o
        return results

    def plan_chains(self, base_tables, chains, favor_min_nodes, max_concurrent=0, want_rows=(), opts=None, net=True):
        """blance_plan_chains: chains of cluster changes, each stage planned on the map the stage before produced.
        chains is a list of chains of equal length; a stage is a dict of SCENARIO_FIELDS and node_in_all ([n_nodes],
        missing = every node; missing scenario keys keep the base's value).  want_rows lists the (chain, stage) pairs
        whose next rows, shapes and warnings are copied out.  opts: None, or one dict of OPT_GROUPS keys per chain.
        Returns (results, nets): results[i][t] a ScenarioResult per stage, nets[i] a ChainNet (None without net)."""
        n = len(chains)
        T = len(chains[0]) if n else 0
        if any(len(c) != T for c in chains):
            raise ValueError("every chain of one call has the same number of stages")
        want = set(want_rows)
        base = base_tables.struct()
        keep, sts = [], (api.ChainStage * max(1, n * T))()
        for i, chain in enumerate(chains):
            for t, stage in enumerate(chain):
                st = sts[i * T + t]
                sc = scenario_tables(base_tables, {k: v for k, v in stage.items() if k != "node_in_all"})
                for f in SCENARIO_FIELDS:
                    v = getattr(sc, f)
                    if f in ("add_is_nil", "has_node_weights"):
                        setattr(st.nodes, f, int(v))
                        continue
                    a = np.ascontiguousarray(v, dtype=np.int32 if f == "node_weight" else np.uint8)
                    keep.append(a)
                    setattr(st.nodes, f, a.ctypes.data if a.size else None)
                m = np.ascontiguousarray(stage.get("node_in_all", np.ones(base_tables.n_nodes)), np.uint8)
                keep.append(m)
                st.node_in_all = m.ctypes.data if m.size else None
        results = [[ScenarioResult(base_tables, (i, t) in want) for t in range(T)] for i in range(n)]
        outs = (api.ScenarioOut * max(1, n * T))(*[r.out for rs in results for r in rs])
        nets = [ChainNet(base_tables) for _ in range(n)] if net else None
        net_arr = (api.ChainOut * max(1, n))(*[x.out for x in nets]) if net else None
        ops = None if opts is None else (api.ScenarioOpts * max(1, n))(*[_opts_struct(base_tables, o, keep) for o in opts])
        self._check(self.lib.blance_plan_chains(self.ptr, ctypes.byref(base), n, T, sts, ops, int(bool(favor_min_nodes)),
                                                int(max_concurrent), outs, net_arr), "blance_plan_chains")
        for i in range(n):
            for t in range(T):
                results[i][t].out = outs[i * T + t]
            if net:
                nets[i].out = net_arr[i]
        return results, nets

    def prepare_batch(self, tables_list, results=None):
        """Builds the blance_plan_in / blance_plan_out arrays of a batch once; run_batch() is then only the
        C call (what a compiled host would do per request)."""
        n = len(tables_list)
        results = results or [PlanResult(t) for t in tables_list]
        ins = (api.PlanIn * n)(*[t.struct() for t in tables_list])
        outs = (api.PlanOut * n)(*[r.out for r in results])
        return n, ins, outs, results, tables_list

    def run_batch(self, prepared):
        n, ins, outs, results, _ = prepared
        self._check(self.lib.blance_plan_next_map_batch(self.ptr, n, ins, outs), "blance_plan_next_map_batch")
        for r, o in zip(results, outs):
            r.out = o
        return results

    def upload(self, tables):
        plan = ctypes.c_void_p()
        s = tables.struct()
        self._check(self.lib.blance_plan_upload(self.ptr, ctypes.byref(s), ctypes.byref(plan)), "blance_plan_upload")
        return plan

    def run(self, plan):
        self._check(self.lib.blance_plan_run(self.ptr, plan), "blance_plan_run")

    def timing(self, plan):
        """(kernel_ms, pass_ms, pass_launches) of the last run()."""
        k, p, n = ctypes.c_float(), ctypes.c_float(), ctypes.c_int32()
        self._check(self.lib.blance_plan_timing(plan, ctypes.byref(k), ctypes.byref(p), ctypes.byref(n)), "blance_plan_timing")
        return k.value, p.value, n.value

    def fetch(self, plan, result):
        self._check(self.lib.blance_plan_fetch(self.ptr, plan, ctypes.byref(result.out)), "blance_plan_fetch")
        return result

    def free(self, plan):
        self.lib.blance_plan_free(self.ptr, plan)

    def calc_partition_moves(self, slot_off, beg_rows, end_rows, favor_min_nodes, n_visit_states=None):
        slot_off = np.ascontiguousarray(slot_off, np.int32)
        beg = np.ascontiguousarray(beg_rows, np.int32)
        end = np.ascontiguousarray(end_rows, np.int32)
        n_states = len(slot_off) - 1
        n_parts = beg.shape[0]
        max_ops = max(1, 2 * int(slot_off[-1]))
        op_node = np.zeros((n_parts, max_ops), np.int32)
        op_state = np.zeros((n_parts, max_ops), np.uint8)
        op_kind = np.zeros((n_parts, max_ops), np.uint8)
        op_count = np.zeros(n_parts, np.int32)
        st = self.lib.blance_calc_partition_moves(
            self.ptr, n_parts, n_states, n_states if n_visit_states is None else n_visit_states, slot_off.ctypes.data,
            beg.ctypes.data, end.ctypes.data, int(bool(favor_min_nodes)), max_ops, op_node.ctypes.data,
            op_state.ctypes.data, op_kind.ctypes.data, op_count.ctypes.data)
        self._check(st, "blance_calc_partition_moves")
        return op_node, op_state, op_kind, op_count

    def moves_create(self, slot_off, beg_rows, end_rows, favor_min_nodes, n_node_ids, n_visit_states=None):
        """blance_moves_create: CalcPartitionMoves of every partition, resident on the device in CSR form.
        Returns (handle, total_ops)."""
        slot_off = np.ascontiguousarray(slot_off, np.int32)
        beg = np.ascontiguousarray(beg_rows, np.int32)
        end = np.ascontiguousarray(end_rows, np.int32)
        n_states = len(slot_off) - 1
        h, tot = ctypes.c_void_p(), ctypes.c_int64()
        st = self.lib.blance_moves_create(self.ptr, beg.shape[0], n_states, n_states if n_visit_states is None else n_visit_states,
                                          slot_off.ctypes.data, beg.ctypes.data, end.ctypes.data, int(bool(favor_min_nodes)),
                                          int(n_node_ids), ctypes.byref(h), ctypes.byref(tot))
        self._check(st, "blance_moves_create")
        return (h, beg.shape[0], int(n_node_ids)), int(tot.value)

    def moves_fetch(self, handle, total_ops):
        h, n_parts, _ = handle
        off = np.zeros(n_parts + 1, np.int64)
        node = np.zeros(max(1, total_ops), np.int32)
        state = np.zeros(max(1, total_ops), np.uint8)
        kind = np.zeros(max(1, total_ops), np.uint8)
        self._check(self.lib.blance_moves_fetch(self.ptr, h, off.ctypes.data, node.ctypes.data, state.ctypes.data, kind.ctypes.data), "blance_moves_fetch")
        return off, node[:total_ops], state[:total_ops], kind[:total_ops]

    def moves_available(self, handle, next_idx):
        h, n_parts, n_node_ids = handle
        nxt = np.ascontiguousarray(next_idx, np.int32)
        node_off = np.zeros(n_node_ids + 1, np.int32)
        node_parts = np.zeros(max(1, n_parts), np.int32)
        best = np.zeros(max(1, n_node_ids), np.int32)
        self._check(self.lib.blance_moves_available(self.ptr, h, nxt.ctypes.data, node_off.ctypes.data, node_parts.ctypes.data, best.ctypes.data),
                    "blance_moves_available")
        return node_off, node_parts[:node_off[-1]], best[:n_node_ids]

    def moves_schedule(self, handle, max_concurrent, node_has_mover=None):
        """blance_moves_schedule + blance_moves_schedule_fetch: the lock-step schedule of the handle's move lists
        (include/blance_b200.h).  Returns (round_off [R+1], sched_op [moves_done], scalars) with scalars a dict of
        rounds, moves_done, stuck_parts, max_batch and device_ms."""
        h, _, n_node_ids = handle
        mover = None if node_has_mover is None else np.ascontiguousarray(node_has_mover, np.uint8)
        if mover is not None and mover.size != n_node_ids:
            raise ValueError("node_has_mover must have n_node_ids = %d entries" % n_node_ids)
        out = api.ScheduleOut()
        self._check(self.lib.blance_moves_schedule(self.ptr, h, int(max_concurrent), None if mover is None else mover.ctypes.data,
                                                   ctypes.byref(out)), "blance_moves_schedule")
        round_off = np.zeros(out.rounds + 1, np.int64)
        sched_op = np.zeros(max(1, out.moves_done), np.int64)
        self._check(self.lib.blance_moves_schedule_fetch(self.ptr, h, round_off.ctypes.data, sched_op.ctypes.data),
                    "blance_moves_schedule_fetch")
        self._rounds[h.value] = out.rounds        # sizes moves_exposure's series
        scalars = {f: getattr(out, f) for f, _ in api.ScheduleOut._fields_}
        return round_off, sched_op[:out.moves_done], scalars

    def moves_exposure(self, handle, constraints, top_state, domain_parent=None, dom=True):
        """blance_moves_exposure: the maps the handle's last moves_schedule passes through, counted per round
        (include/blance_b200.h); its R sizes the series.  Returns a dict:
        series [6][R + 1], peak / peak_round / area [6] (abi.EXPO_METRICS order), dom_peak / dom_peak_round [V],
        part_min_copies / part_no_top / part_flags [n_parts], rounds and kernel_ms.  dom=False asks for no dom_peak
        (its arrays are then zero)."""
        h, n_parts, n_node_ids = handle
        keep = []
        cons = np.ascontiguousarray(constraints, np.int32)
        e_in = api.ExposureIn(cons.ctypes.data if cons.size else None, int(top_state), 0, None)
        V = n_node_ids
        if domain_parent is not None:
            par = np.ascontiguousarray(domain_parent, np.int32)
            keep.append(par)
            e_in.n_domains = par.size - n_node_ids
            e_in.domain_parent = par.ctypes.data
            V = par.size
        rounds = self._rounds.get(h.value)
        if rounds is None:                      # not scheduled through this context: the library refuses the handle
            self._check(self.lib.blance_moves_exposure(self.ptr, h, ctypes.byref(e_in), ctypes.byref(api.ExposureOut())),
                        "blance_moves_exposure")
            raise ValueError("schedule the handle with moves_schedule before moves_exposure")
        res = dict(series=np.zeros((6, rounds + 1), np.int64), dom_peak=np.zeros(max(1, V), np.int64),
                   dom_peak_round=np.zeros(max(1, V), np.int32), part_min_copies=np.zeros(max(1, n_parts), np.int32),
                   part_no_top=np.zeros(max(1, n_parts), np.int32), part_flags=np.zeros(max(1, n_parts), np.uint8))
        out = api.ExposureOut()
        for k, a in res.items():
            setattr(out, k, a.ctypes.data if dom or not k.startswith("dom") else None)
        self._check(self.lib.blance_moves_exposure(self.ptr, h, ctypes.byref(e_in), ctypes.byref(out)), "blance_moves_exposure")
        for k in ("dom_peak", "dom_peak_round"):
            res[k] = res[k][:V]
        for k in ("part_min_copies", "part_no_top", "part_flags"):
            res[k] = res[k][:n_parts]
        res.update(rounds=out.rounds, kernel_ms=out.kernel_ms, peak=np.array(out.peak[:], np.int64),
                   peak_round=np.array(out.peak_round[:], np.int32), area=np.array(out.area[:], np.int64))
        return res

    def moves_free(self, handle):
        self._rounds.pop(handle[0].value, None)
        self.lib.blance_moves_free(self.ptr, handle[0])

    def kernel_launches(self):
        return int(self.lib.blance_ctx_kernel_launches(self.ptr))

    def close(self):
        if self.ptr:
            self.lib.blance_ctx_destroy(self.ptr)
            self.ptr = ctypes.c_void_p()
