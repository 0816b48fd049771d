"""Two readings of each node's load while a rebalance runs (blance_moves_load, include/blance_b200.h), sharing no code
with the product or with each other:

  replay()      the literal one: every partition a list of (node, state) entries, each round's ops applied as the
                reference's test app applies an AssignPartitionsFunc call (orchestrate_test.go:137-157), and load_t
                counted on every map M_0 .. M_R;
  vectorised()  numpy over per-entry intervals [start, end) of rounds, for inputs far too large to replay map by map.

Both take the handle's tables as the tests fetch them: slot_off, beg rows, the CSR ops (op_off, op_node, op_state,
op_kind), the schedule (round_off [R + 1], sched_op), n_node_ids and the weights w [n_parts] (None: every partition
weighs 1).  They return the dict Context.moves_load returns (without kernel_ms)."""
import numpy as np

from exposure_oracle import beg_entries

DEL = 1


def _result(load, S, NU):
    """load [R + 1][S + 1][NU] or the per-key series -> the outputs."""
    beg, end = load[0], load[-1]
    peak = load.max(axis=0)
    peak_round = np.argmax(load == peak[None], axis=0).astype(np.int32)
    if NU:
        over = peak[S] - np.maximum(beg[S], end[S])
        over_max, over_node = int(over.max()), int(np.argmax(over))
    else:
        over_max, over_node = 0, -1
    return dict(rounds=load.shape[0] - 1, node_beg=beg, node_end=end, node_peak=peak, node_peak_round=peak_round,
                over_max=over_max, over_node=over_node)


def replay(slot_off, beg, op_off, op_node, op_state, op_kind, round_off, sched_op, n_node_ids, w=None):
    S = len(slot_off) - 1
    P = len(op_off) - 1
    R = len(round_off) - 1
    NU = n_node_ids
    w = [1] * P if w is None else [int(x) for x in w]
    maps = [beg_entries(slot_off, beg[p]) for p in range(P)]
    part_of = np.searchsorted(op_off, np.arange(int(op_off[-1])), side="right") - 1
    load = np.zeros((R + 1, S + 1, NU), np.int64)
    for t in range(R + 1):
        if t > 0:
            for i in sched_op[round_off[t - 1]:round_off[t]]:
                p, n = int(part_of[i]), int(op_node[i])
                maps[p] = [e for e in maps[p] if e[0] != n]
                if op_kind[i] != DEL:
                    maps[p].append((n, int(op_state[i])))
        for p in range(P):
            for n, s in maps[p]:
                if 0 <= n < NU:
                    load[t, s, n] += w[p]
                    load[t, S, n] += w[p]
    return _result(load, S, NU)


def vectorised(slot_off, beg, op_off, op_node, op_state, op_kind, round_off, sched_op, n_node_ids, w=None):
    slot_off = np.asarray(slot_off, np.int64)
    beg = np.asarray(beg, np.int64).reshape(len(op_off) - 1, int(slot_off[-1]))
    op_off = np.asarray(op_off, np.int64)
    op_node = np.asarray(op_node, np.int64)
    S, P, R, NU = len(slot_off) - 1, len(op_off) - 1, len(round_off) - 1, n_node_ids
    SL = int(slot_off[-1])
    w = np.ones(P, np.int64) if w is None else np.asarray(w, np.int64)
    T = int(op_off[-1])
    # the round each op is applied at the end of (-1: never), and its partition
    rho = np.full(T, -1, np.int64)
    ro = np.asarray(round_off, np.int64)
    if len(sched_op):
        rho[np.asarray(sched_op, np.int64)] = np.searchsorted(ro, np.arange(len(sched_op)), side="right") - 1
    part = np.repeat(np.arange(P), np.diff(op_off))
    applied = rho >= 0
    # beg entries: the slots of a state before its first -1; each lives until its node's op is applied
    state_of = np.searchsorted(slot_off, np.arange(SL), side="right") - 1
    empty = beg == -1
    closed = np.zeros_like(empty)
    for s in range(S):
        a, b = int(slot_off[s]), int(slot_off[s + 1])
        if b > a:
            closed[:, a:b] = np.cumsum(empty[:, a:b], axis=1) > 0
    pp, xx = np.nonzero(~closed)
    bn, bs = beg[pp, xx], state_of[xx]
    # the op of (p, node), if applied: its round ends the entry
    big = int(max(NU, int(op_node.max(initial=0)) + 1, int(beg.max(initial=0)) + 1)) + 1
    okey = part[applied] * big + op_node[applied]
    order = np.argsort(okey, kind="stable")
    okey, orho = okey[order], rho[applied][order]
    bkey = pp * big + bn
    j = np.searchsorted(okey, bkey)
    hit = (j < len(okey)) & (okey[np.minimum(j, max(len(okey) - 1, 0))] == bkey) if len(okey) else np.zeros(len(bkey), bool)
    b_end = np.where(hit, orho[np.minimum(j, max(len(okey) - 1, 0))] + 1 if len(okey) else 0, R + 1)
    # entries added by applied ops that are not dels: from rho + 1 to the end
    add = applied & (np.asarray(op_kind) != DEL)
    nodes = np.concatenate([bn, op_node[add]])
    states = np.concatenate([bs, np.asarray(op_state, np.int64)[add]])
    start = np.concatenate([np.zeros(len(bn), np.int64), rho[add] + 1])
    stop = np.concatenate([b_end, np.full(int(add.sum()), R + 1, np.int64)])
    wt = np.concatenate([w[pp], w[part[add]]])
    keep = (nodes >= 0) & (nodes < NU) & (start < stop)
    nodes, states, start, stop, wt = nodes[keep], states[keep], start[keep], stop[keep], wt[keep]
    diff = np.zeros((R + 2, S + 1, NU), np.int64)
    for s_idx in (states, np.full(len(states), S)):
        np.add.at(diff, (start, s_idx, nodes), wt)
        np.add.at(diff, (stop, s_idx, nodes), -wt)
    return _result(np.cumsum(diff, axis=0)[:R + 1], S, NU)


def assert_equal(got, want, where=None):
    for k in ("rounds", "over_max", "over_node"):
        assert got[k] == want[k], (where, k, got[k], want[k])
    for k in ("node_beg", "node_end", "node_peak", "node_peak_round"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), (where, k)
