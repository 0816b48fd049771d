"""Two readings of the exposure of a rebalance (blance_moves_exposure, include/blance_b200.h), sharing no code with
the product or with each other:

  replay()      the literal one: every partition a list of (node, state) entries, each round's ops applied as the
                reference's test app applies an AssignPartitionsFunc call (orchestrate_test.go:137-157), and every
                metric counted on every map M_0 .. M_R;
  vectorised()  numpy over per-op intervals, for inputs far too large to replay map by map.

Both take the handle's tables as the tests fetch them: slot_off, beg rows, the CSR ops (op_off, op_node, op_state,
op_kind), the schedule (round_off [R + 1], sched_op), constraints, top_state, n_node_ids and optionally the
fault-domain forest domain_parent [n_node_ids + n_domains].  They return the dict Context.moves_exposure returns
(without kernel_ms)."""
import numpy as np

METRICS = ("NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY", "COPIES")
DEL = 1


def beg_entries(slot_off, row):
    """(node, state) entries of one row: each state's slots before its first -1."""
    out = []
    for s in range(len(slot_off) - 1):
        for i in range(slot_off[s], slot_off[s + 1]):
            if row[i] == -1:
                break
            out.append((int(row[i]), s))
    return out


def _values(entries, S, cons, top):
    c = [0] * S
    for _, s in entries:
        c[s] += 1
    C = len(entries)
    return (int(top >= 0 and c[top] == 0),
            int(top >= 0 and cons[top] > 0 and c[top] > cons[top]),
            int(any(cons[s] > 0 and c[s] < cons[s] for s in range(S))),
            int(C == 1), int(C == 0), C)


def _ancestors(v, parent):
    out = []
    while v >= 0:
        out.append(v)
        v = -1 if parent is None else int(parent[v])
    return out


def replay(slot_off, beg, op_off, op_node, op_state, op_kind, round_off, sched_op, constraints, top_state, n_node_ids,
           domain_parent=None):
    S = len(slot_off) - 1
    P = len(op_off) - 1
    R = len(round_off) - 1
    V = n_node_ids if domain_parent is None else len(domain_parent)
    maps = [beg_entries(slot_off, beg[p]) for p in range(P)]
    part_of = np.searchsorted(op_off, np.arange(int(op_off[-1])), side="right") - 1
    series = np.zeros((6, R + 1), np.int64)
    dom_cnt = np.zeros((R + 1, V), np.int64)
    min_c = [None] * P
    no_top = [0] * P
    flags = [0] * P
    for t in range(R + 1):
        if t > 0:
            for i in sched_op[round_off[t - 1]:round_off[t]]:
                p, n = int(part_of[i]), int(op_node[i])
                maps[p] = [e for e in maps[p] if e[0] != n]
                if op_kind[i] != DEL:
                    maps[p].append((n, int(op_state[i])))
        for p in range(P):
            v = _values(maps[p], S, constraints, top_state)
            for m in range(6):
                series[m, t] += v[m]
                flags[p] |= (v[m] != 0) << m
            min_c[p] = v[5] if min_c[p] is None else min(min_c[p], v[5])
            no_top[p] += v[0]
            if maps[p] and all(0 <= n < n_node_ids for n, _ in maps[p]):
                common = None
                for n, _ in maps[p]:
                    a = set(_ancestors(n, domain_parent))
                    common = a if common is None else common & a
                for x in common:
                    dom_cnt[t, x] += 1
    peak = series.max(axis=1)
    return dict(rounds=R, series=series, peak=peak, peak_round=np.argmax(series == peak[:, None], axis=1).astype(np.int32),
                area=series.sum(axis=1), dom_peak=dom_cnt.max(axis=0) if V else np.zeros(0, np.int64),
                dom_peak_round=np.argmax(dom_cnt == dom_cnt.max(axis=0), axis=0).astype(np.int32) if V else np.zeros(0, np.int32),
                part_min_copies=np.asarray(min_c, np.int32), part_no_top=np.asarray(no_top, np.int32),
                part_flags=np.asarray(flags, np.uint8))


def _paths(n_node_ids, parent):
    """[V + 1, 17]: each vertex's chain to its root, padded with -1; row V (index -1) is the empty chain."""
    V = n_node_ids if parent is None else len(parent)
    out = np.full((V + 1, 17), -1, np.int64)
    out[:V, 0] = np.arange(V)
    if parent is not None:
        par = np.append(np.asarray(parent, np.int64), -1)
        for d in range(1, 17):
            out[:V, d] = np.where(out[:V, d - 1] >= 0, par[out[:V, d - 1]], -1)
    return out


def _dca(nodes, n_node_ids, paths):
    """Deepest common ancestor of each row of nodes [P, K] (-1 = no entry; another id outside [0, n_node_ids) lies
    under no vertex); -1 when there is none."""
    P, K = nodes.shape
    has = nodes != -1
    bad = (has & ((nodes < 0) | (nodes >= n_node_ids))).any(axis=1) | ~has.any(axis=1)
    nd = np.where(has & ~bad[:, None], nodes, -1)
    if paths is None:                                            # every node its own root: one node or none
        first = nd[np.arange(P), np.argmax(nd >= 0, axis=1)] if K else np.full(P, -1)
        one = ((nd == first[:, None]) | (nd < 0)).all(axis=1)
        return np.where(bad | ~one, -1, first)
    # root-first chains, right-aligned by depth so that equal prefixes line up
    ch = paths[nd]                                               # [P, K, 17] leaf first
    depth = (ch >= 0).sum(axis=2)
    maxd = 17
    idx = depth[:, :, None] - 1 - np.arange(maxd)[None, None, :]  # root-first position d -> leaf-first index
    rf = np.where(idx >= 0, np.take_along_axis(ch, np.clip(idx, 0, 16), axis=2), -2)
    first = np.argmax(nd >= 0, axis=1)
    ref = rf[np.arange(P), first]                                # [P, 17]
    same = np.where((nd >= 0)[:, :, None], rf == ref[:, None, :], True).all(axis=1) & (ref >= 0)
    L = np.cumprod(same, axis=1).sum(axis=1)
    d = np.where(L > 0, ref[np.arange(P), np.maximum(L - 1, 0)], -1)
    return np.where(bad, -1, d)


def vectorised(slot_off, beg, op_off, op_node, op_state, op_kind, round_off, sched_op, constraints, top_state, n_node_ids,
               domain_parent=None):
    slot_off = np.asarray(slot_off, np.int64)
    beg = np.asarray(beg, np.int64).reshape(len(op_off) - 1, int(slot_off[-1]))
    op_off = np.asarray(op_off, np.int64)
    S, P, R = len(slot_off) - 1, len(op_off) - 1, len(round_off) - 1
    SL = int(slot_off[-1])
    cons = np.asarray(constraints, np.int64)
    V = n_node_ids if domain_parent is None else len(domain_parent)
    T = int(op_off[-1])
    op_round = np.full(T, -1, np.int64)
    op_round[np.asarray(sched_op, np.int64)] = np.repeat(np.arange(R), np.diff(np.asarray(round_off, np.int64)))
    slot_state = np.searchsorted(slot_off, np.arange(SL), side="right") - 1
    # entries: slots before each state's first -1
    live = beg != -1
    for s in range(S):
        lo, hi = slot_off[s], slot_off[s + 1]
        if hi > lo:
            live[:, lo:hi] = np.cumprod(live[:, lo:hi], axis=1).astype(bool)
    c = np.zeros((P, max(S, 1)), np.int64)
    for i in range(SL):
        c[:, slot_state[i]] += live[:, i]

    def values(c):
        C = c[:, :S].sum(axis=1)
        ctop = c[:, top_state] if top_state >= 0 else np.zeros(P, np.int64)
        ktop = cons[top_state] if top_state >= 0 else 0
        short = np.zeros(P, bool)
        for s in range(S):
            if cons[s] > 0:
                short |= c[:, s] < cons[s]
        return np.stack([(top_state >= 0) & (ctop == 0), (top_state >= 0) & (ktop > 0) & (ctop > ktop), short,
                         C == 1, C == 0, C]).astype(np.int64)

    paths = _paths(n_node_ids, domain_parent)
    n_ops = np.diff(op_off)
    J = int(n_ops.max()) if P else 0
    added = np.full((P, max(J, 1)), -1, np.int64)

    def dca(ps=slice(None)):
        return _dca(np.concatenate([np.where(live[ps], beg[ps], -1), added[ps]], axis=1), n_node_ids,
                    None if domain_parent is None else paths)

    diff = np.zeros((6, R + 2), np.int64)
    v = values(c)
    diff[:, 0] = v.sum(axis=1)
    flags = np.zeros(P, np.int64)
    for m in range(6):
        flags |= (v[m] != 0).astype(np.int64) << m
    min_c = v[5].copy()
    no_top = np.zeros(P, np.int64)
    t0 = np.zeros(P, np.int64)
    d_prev = dca()
    base = np.zeros(V + 1, np.int64)
    np.add.at(base, paths[d_prev][d_prev >= 0].ravel(), 1)
    ev_v, ev_t, ev_d = [], [], []
    alive = np.ones(P, bool)
    for j in range(J):
        k = op_off[:-1] + j
        sel = alive & (n_ops > j)
        sel[sel] = op_round[k[sel]] >= 0
        alive = sel
        if not sel.any():
            break
        ps = np.nonzero(sel)[0]
        ks = k[ps]
        r = op_round[ks]
        n = np.asarray(op_node, np.int64)[ks]
        no_top[ps] += v[0, ps] * (r + 1 - t0[ps])
        t0[ps] = r + 1
        for i in range(SL):
            hit = live[ps, i] & (beg[ps, i] == n)
            c[ps[hit], slot_state[i]] -= 1
            live[ps[hit], i] = False
        notdel = np.asarray(op_kind, np.int64)[ks] != DEL
        st = np.asarray(op_state, np.int64)[ks]
        c[ps[notdel], st[notdel]] += 1
        added[ps[notdel], j] = n[notdel]
        u = values(c)
        for m in range(6):
            np.add.at(diff[m], r + 1, (u[m] - v[m])[ps])
            flags[ps] |= (u[m, ps] != 0).astype(np.int64) << m
        v = u
        min_c = np.minimum(min_c, v[5])
        d = d_prev.copy()
        d[ps] = dca(ps)
        ch = ps[d[ps] != d_prev[ps]]
        for dd, sign in ((d_prev[ch], -1), (d[ch], 1)):
            chains = paths[dd]                                      # full chains: the common part cancels per (v, t)
            ok = (chains >= 0) & (dd >= 0)[:, None]
            ev_v.append(chains[ok])
            ev_t.append(np.broadcast_to((op_round[op_off[ch] + j] + 1)[:, None], chains.shape)[ok])
            ev_d.append(np.full(int(ok.sum()), sign, np.int64))
        d_prev = d
    no_top += v[0] * (R + 1 - t0)
    series = np.cumsum(diff[:, :R + 1], axis=1)
    peak = series.max(axis=1)
    dom_peak, dom_round = base[:V].copy(), np.zeros(V, np.int64)
    if ev_v:
        ev_v, ev_t, ev_d = np.concatenate(ev_v), np.concatenate(ev_t), np.concatenate(ev_d)
        if ev_v.size:
            key = ev_v * (R + 2) + ev_t
            uk, inv = np.unique(key, return_inverse=True)
            tot = np.zeros(uk.size, np.int64)
            np.add.at(tot, inv, ev_d)
            uv, ut = uk // (R + 2), uk % (R + 2)
            cs = np.cumsum(tot)
            start = np.searchsorted(uv, uv, side="left")
            run = cs - np.where(start > 0, cs[start - 1], 0)
            cnt = base[uv] + run
            order = np.lexsort((ut, -cnt, uv))
            first = order[np.r_[True, uv[order][1:] != uv[order][:-1]]]
            better = cnt[first] > dom_peak[uv[first]]
            dom_peak[uv[first][better]] = cnt[first][better]
            dom_round[uv[first][better]] = ut[first][better]
    return dict(rounds=R, series=series, peak=peak, peak_round=np.argmax(series == peak[:, None], axis=1).astype(np.int32),
                area=series.sum(axis=1), dom_peak=dom_peak, dom_peak_round=dom_round.astype(np.int32),
                part_min_copies=min_c.astype(np.int32), part_no_top=no_top.astype(np.int32), part_flags=flags.astype(np.uint8))


def assert_equal(got, want, what=""):
    for k in ("rounds", "series", "peak", "peak_round", "area", "dom_peak", "dom_peak_round", "part_min_copies",
              "part_no_top", "part_flags"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), (what, k, got[k], want[k])
