"""The chain reference of blance_plan_chains, built from the CPU oracle (oracle/fast.c): every stage is planned as
one plain PlanNextMapEx instance.  Stage t's tables follow the chain rule of include/blance_b200.h from stage t-1's
next rows; its node ids are RENUMBERED so that the members of nodesAll_t come first, in universe order, and the
universe's other ids follow - the single-plan form, with no membership mask.  The oracle's rows are mapped back to the
chain's ids, and the summaries are recomputed as for scenarios (test_scenarios_gpu.reference_summary)."""
import copy
import ctypes

import numpy as np

from oracle_loader import fast_lib_path
from test_scenarios_gpu import reference_summary

from blance_b200 import abi, tables

FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]

STAGE_KEYS = tables.SCENARIO_FIELDS + ("node_in_all",)


def _array(ptr, ctype, n, dtype):
    if not ptr or n <= 0:
        return np.zeros(max(n, 0), dtype)
    return np.ctypeslib.as_array((ctype * n).from_address(ptr)).astype(dtype).copy()


def tables_from_struct(s):
    """PlanTables holding copies of every array of the blance_plan_in `s` (e.g. an interned plan's)."""
    S, P, N, NU, SL = s.n_states, s.n_parts, s.n_nodes, s.n_node_ids, s.n_slots
    t = tables.PlanTables(N, S, P, [0] * S, [0] * S, n_node_ids=NU)
    for f in abi._I32_FIELDS:
        setattr(t, f, int(getattr(s, f)))
    t.n_rules, t.n_hier_bits, t.engine = int(s.n_rules), int(s.n_hier_bits), int(s.engine)
    i32, u8 = ctypes.c_int32, ctypes.c_uint8
    for f, n in (("state_priority", S), ("state_constraints", S), ("state_slot_off", S + 1), ("state_stickiness", S),
                 ("node_weight", N), ("part_weight", P), ("part_name_rank", P), ("extra_tot_first", N),
                 ("extra_tot_rest", N)):
        setattr(t, f, _array(getattr(s, f), i32, n, np.int32))
    for f, n in (("state_has_stickiness", S), ("node_removed", NU), ("node_added", NU), ("node_has_weight", N),
                 ("part_in_prev", P), ("part_in_assign", P), ("part_has_weight", P)):
        setattr(t, f, _array(getattr(s, f), u8, n, np.uint8))
    t.prev_rows = _array(s.prev_rows, i32, P * SL, np.int32).reshape(P, SL)
    t.cur_rows = _array(s.cur_rows, i32, P * SL, np.int32).reshape(P, SL)
    t.prev_shape = _array(s.prev_shape, u8, P * S, np.uint8).reshape(P, S)
    t.cur_shape = _array(s.cur_shape, u8, P * S, np.uint8).reshape(P, S)
    t.rule_off = _array(s.rule_off, i32, S + 1, np.int32) if s.has_hier_rules else np.zeros(S + 1, np.int32)
    words = s.n_rules * (NU + 1) * ((s.n_hier_bits + 31) // 32) if s.has_hier_rules else 0
    t.ie_mask = _array(s.ie_mask, ctypes.c_uint32, words, np.uint32)
    return t


def stage_fields(s):
    """The six node fields of the blance_plan_in `s`, as a stage dict."""
    t = tables_from_struct(s)
    return {f: copy.deepcopy(getattr(t, f)) for f in tables.SCENARIO_FIELDS}


def substituted(cur, stage, opts, t):
    """Stage t's instance in chain ids: `cur` (the partition tables as the chain rule left them) with the stage's node
    fields and the chain's options; from stage 2 on the non-model counts of iteration 1 are extra_tot_rest."""
    x = tables.scenario_tables(cur, {k: v for k, v in stage.items() if k != "node_in_all"}, opts)
    x.node_removed = (np.asarray(x.node_removed) != 0).astype(np.uint8)
    if t > 0:
        x.extra_tot_first = np.array(x.extra_tot_rest, np.int32)
    return x


def renumbered(x, node_in_all):
    """x with the members of nodesAll first (universe order): returns (tables, order) where order[new id] = chain id."""
    N, NU = x.n_nodes, x.n_node_ids
    inall = np.asarray(node_in_all, bool) if node_in_all is not None else np.ones(N, bool)
    members = np.flatnonzero(inall)
    order = np.concatenate([members, np.flatnonzero(~inall), np.arange(N, NU)]).astype(np.int64)
    new_of = np.empty(NU, np.int64)
    new_of[order] = np.arange(NU)
    r = copy.copy(x)
    r.n_nodes = int(members.size)
    for f in ("prev_rows", "cur_rows"):
        rows = np.asarray(getattr(x, f))
        setattr(r, f, np.where(rows >= 0, new_of[np.maximum(rows, 0)], -1).astype(np.int32))
    r.node_removed = np.asarray(x.node_removed, np.uint8)[order]
    r.node_added = np.asarray(x.node_added, np.uint8)[order]
    for f in ("node_weight", "node_has_weight", "extra_tot_first", "extra_tot_rest"):
        setattr(r, f, np.asarray(getattr(x, f))[members])
    if x.has_hier_rules and x.n_rules > 0:
        HW = (x.n_hier_bits + 31) // 32
        m = np.asarray(x.ie_mask, np.uint32).reshape(x.n_rules, NU + 1, HW)
        bits = np.unpackbits(m.view(np.uint8).reshape(x.n_rules, NU + 1, HW * 4), axis=2, bitorder="little")
        anchor = np.concatenate([order, [NU]])                    # new anchor a' holds old anchor anchor[a']
        bits = bits[:, anchor, :]
        col = np.arange(bits.shape[2])
        src = col.copy()                                         # new bit b' holds old bit src[b']
        src[:N] = order[:N]
        bits = bits[:, :, src]
        packed = np.ascontiguousarray(np.packbits(np.ascontiguousarray(bits), axis=2, bitorder="little"))
        r.ie_mask = packed.view(np.uint32).reshape(-1).copy()
    return r, order


def oracle(t):
    r = tables.PlanResult(t)
    s = t.struct()
    assert FAST.oracle_fast_plan_next_map(ctypes.byref(s), ctypes.byref(r.out)) == 0
    return r


def advance(cur, next_rows, next_shape):
    """The chain rule: the partition tables of the next stage."""
    a = np.asarray(cur.part_in_assign) != 0
    c = copy.copy(cur)
    c.prev_rows = np.where(a[:, None], next_rows, cur.prev_rows).astype(np.int32)
    c.cur_rows = np.where(a[:, None], next_rows, cur.cur_rows).astype(np.int32)
    c.prev_shape = np.where(a[:, None], next_shape, cur.prev_shape).astype(np.uint8)
    c.cur_shape = np.where(a[:, None], next_shape, cur.cur_shape).astype(np.uint8)
    c.part_in_prev = np.where(a, 1, cur.part_in_prev).astype(np.uint8)
    return c


def chain_reference(base, chain, opts=None, favor_min_nodes=False):
    """The per-stage results of one chain (a list of stage dicts of STAGE_KEYS) over PlanTables `base`, and its net
    summary.  Returns (stages, net): each stage a dict of next_rows, next_shape, warn, iters_run, converged, steps and
    the summaries; net a dict of node_ops, ops_total and parts_moved."""
    cur, out = base, []
    for t, stage in enumerate(chain):
        x = substituted(cur, stage, opts, t)
        r, order = renumbered(x, stage.get("node_in_all"))
        ref = oracle(r)
        nxt = np.where(ref.next_rows >= 0, order[np.maximum(ref.next_rows, 0)], -1).astype(np.int32)
        res = dict(next_rows=nxt, next_shape=ref.next_shape.copy(), warn=ref.warn.copy(), iters_run=ref.iters_run,
                   converged=ref.converged, steps=ref.steps)
        res.update(reference_summary(x, nxt, ref.warn, favor_min_nodes))
        out.append(res)
        cur = advance(cur, nxt, ref.next_shape)
    # the base's prev rows as the beg rows: of that summary only the moves are read
    s = reference_summary(substituted(base, chain[-1], opts, 0), out[-1]["next_rows"], out[-1]["warn"], favor_min_nodes)
    return out, dict(node_ops=s["node_ops"], ops_total=s["ops_total"], parts_moved=s["parts_moved"])


STAGE_FIELDS = ("next_rows", "next_shape", "warn", "node_ops", "state_node_load")
STAGE_SCALARS = ("iters_run", "converged", "steps", "parts_moved", "ops_total", "warn_parts")


def assert_stage(got, ref, what):
    """A ScenarioResult (rows copied out) against a stage of chain_reference."""
    for f in STAGE_FIELDS:
        assert np.array_equal(getattr(got, f), ref[f]), (what, f)
    for f in STAGE_SCALARS:
        assert getattr(got, f) == ref[f], (what, f, getattr(got, f), ref[f])
