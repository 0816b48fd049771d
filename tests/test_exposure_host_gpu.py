"""blance_b200.OrchestrateExposure over string maps: equal to a literal replay of OrchestrateSchedule's batches, as
the reference's test app applies AssignPartitionsFunc calls (orchestrate_test.go:137-157), with and without a
NodeHierarchy.  Needs an H100; run with -m gpu."""
import random

import pytest

import blance_b200

pytestmark = pytest.mark.gpu
METRICS = ("NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY", "COPIES")


def replay(model, begMap, rounds, hierarchy):
    """The exposure of `rounds` (OrchestrateSchedule's batches) over the string map begMap, keyed as
    OrchestrateExposure keys it."""
    top = min(sorted(model), key=lambda s: model[s][0]) if model else None
    maps = {p: [(n, s) for s, lst in nbs.items() for n in (lst or [])] for p, nbs in begMap.items()}

    def ancestors(n):
        out = [n]
        while hierarchy and hierarchy.get(out[-1], ""):
            out.append(hierarchy[out[-1]])
        return out

    series = {m: [] for m in METRICS}
    dom, part = [], {p: [] for p in maps}
    for t in range(len(rounds) + 1):
        if t:
            for call in rounds[t - 1]:
                for p, s in zip(call.Partitions, call.States):
                    maps[p] = [e for e in maps[p] if e[0] != call.Node] + ([(call.Node, s)] if s else [])
        cnt, dcount = {m: 0 for m in METRICS}, {}
        for p, ents in maps.items():
            c = {}
            for _, s in ents:
                c[s] = c.get(s, 0) + 1
            k_top = model[top][1] if top else 0
            v = dict(NO_TOP=int(top is not None and c.get(top, 0) == 0),
                     MULTI_TOP=int(top is not None and k_top > 0 and c.get(top, 0) > k_top),
                     SHORT=int(any(k > 0 and c.get(s, 0) < k for s, (_, k) in model.items())),
                     ONE_COPY=int(len(ents) == 1), NO_COPY=int(not ents), COPIES=len(ents))
            for m in METRICS:
                cnt[m] += v[m]
            part[p].append(v)
            if ents:
                common = set(ancestors(ents[0][0]))
                for n, _ in ents[1:]:
                    common &= set(ancestors(n))
                for x in common:
                    dcount[x] = dcount.get(x, 0) + 1
        for m in METRICS:
            series[m].append(cnt[m])
        dom.append(dcount)
    res = dict(rounds=len(rounds), series=series, peak={m: max(series[m]) for m in METRICS},
               peak_round={m: series[m].index(max(series[m])) for m in METRICS}, area={m: sum(series[m]) for m in METRICS})
    names = {x for d in dom for x in d}
    res["dom_peak"] = {x: max(d.get(x, 0) for d in dom) for x in names}
    res["dom_peak_round"] = {x: [d.get(x, 0) for d in dom].index(res["dom_peak"][x]) for x in names}
    res["part_min_copies"] = {p: min(v["COPIES"] for v in vs) for p, vs in part.items()}
    res["part_no_top"] = {p: sum(v["NO_TOP"] for v in vs) for p, vs in part.items()}
    res["part_flags"] = {p: sum(1 << i for i, m in enumerate(METRICS) if any(v[m] for v in vs)) for p, vs in part.items()}
    for k in ("dom_peak", "dom_peak_round", "part_min_copies", "part_no_top", "part_flags"):
        keep = res["dom_peak"] if k == "dom_peak_round" else res[k]
        res[k] = {x: y for x, y in res[k].items() if keep[x]}
    return res


def random_maps(rnd, nodes, states, P):
    def side():
        m = {}
        for p in range(P):
            avail = nodes[:]
            rnd.shuffle(avail)
            nbs = {}
            for s in states:
                if rnd.random() < 0.2:
                    continue
                nbs[s] = [avail.pop() for _ in range(rnd.randint(0, 2))]
            m["p%03d" % p] = nbs
        return m
    beg, end = side(), side()
    for p in rnd.sample(sorted(beg), P // 6):
        end[p] = {k: list(v) for k, v in beg[p].items()}
    return beg, end


def check(model, nodesAll, beg, end, conc, favor, hierarchy=None):
    opts = blance_b200.OrchestratorOptions(MaxConcurrentPartitionMovesPerNode=conc, FavorMinNodes=favor)
    got = blance_b200.OrchestrateExposure(model, opts, nodesAll, beg, end, hierarchy)
    rounds = blance_b200.OrchestrateSchedule(model, opts, nodesAll, beg, end)
    want = replay(model, beg, rounds, hierarchy)
    for k in want:
        g = got[k]
        if k == "series":
            g = {m: list(v) for m, v in g.items()}
        assert g == want[k], (k, conc, favor)
    return got


def test_primary_move_both_ways():
    model = {"primary": (0, 1), "replica": (1, 1)}
    beg = {"p": {"primary": ["a"]}}
    end = {"p": {"primary": ["b"]}}
    no_copy = check(model, ["a", "b"], beg, end, 1, True)
    two = check(model, ["a", "b"], beg, end, 1, False)
    assert no_copy["series"]["NO_COPY"] == [0, 1, 0] and no_copy["part_min_copies"] == {}
    assert two["series"]["MULTI_TOP"] == [0, 1, 0] and two["part_min_copies"] == {"p": 1}


@pytest.mark.parametrize("seed", range(6))
def test_random_string_maps_equal_the_replay(seed):
    rnd = random.Random(seed)
    nodes = ["n%d" % i for i in range(7)]
    model = {"primary": (0, 1), "replica": (1, 2)} if seed % 2 else {"primary": (0, 1), "replica": (1, 1), "zz": (0, 0)}
    beg, end = random_maps(rnd, nodes, sorted(model), 40)
    nodesAll = nodes if seed % 3 else nodes[:-1]          # the last node without a mover: stuck partitions
    hierarchy = None
    if seed >= 3:                                         # racks under two zones, one node outside the hierarchy
        hierarchy = {n: "rack%d" % (i % 3) for i, n in enumerate(nodes[:-1])}
        hierarchy.update({"rack0": "zoneA", "rack1": "zoneA", "rack2": "zoneB"})
    for conc in (1, 2, 4):
        for favor in (False, True):
            check(model, nodesAll, beg, end, conc, favor, hierarchy)


def test_mismatched_maps_and_unsupported_states():
    with pytest.raises(blance_b200.BlanceError, match="mismatched begMap and endMap"):
        blance_b200.OrchestrateExposure({"primary": (0, 1)}, None, ["a"], {"0": {"primary": ["a"]}}, {})
    states = {"s%d" % i: (i, 1) for i in range(9)}
    m = {"0": {s: ["n%d" % i] for i, s in enumerate(states)}}
    with pytest.raises(blance_b200.BlanceError, match="more than 8 states"):
        blance_b200.OrchestrateExposure(states, None, ["a"], m, m)

