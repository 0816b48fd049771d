"""blance_b200.PlanNextMapScenarios(..., exposure) over string maps: every scenario's exposure at every count equals
OrchestrateExposure(model with the scenario's constraints, {c, favorMinNodes}, nodesAll, begMap, finalMap,
NodeHierarchy), with begMap = prevMap plus an empty entry for every assigned partition it lacks and finalMap = prevMap
with the assigned partitions' next rows.  Names are fixed-width, so interning order equals byte order (the one
documented difference to the schedule twin).  Needs an H100; run with -m gpu."""
import random

import pytest

import blance_b200

pytestmark = pytest.mark.gpu
NODES = ["n%02d" % i for i in range(12)]
HIERARCHY = dict({n: "rack%d" % (i % 4) for i, n in enumerate(NODES[:-1])}, rack0="zoneA", rack1="zoneA", rack2="zoneB", rack3="zoneB")


def prev_map(rnd, P, states=("primary", "replica")):
    out = {}
    for p in range(P):
        a = rnd.sample(NODES, 3)
        out["p%03d" % p] = {"primary": [a[0]], "replica": a[1:1 + rnd.randint(0, 2)]} if len(states) == 2 else {"primary": [a[0]]}
    return out


def check(prev, assign, model, scs, counts, favor, hierarchy, cap=4096):
    opts = blance_b200.PlanNextMapOptions(NodeHierarchy=hierarchy)
    res = blance_b200.PlanNextMapScenarios(prev, assign, NODES, model, opts, scs, favor, wantMaps=range(len(scs)),
                                           scheduleConcurrency=counts, exposure={"seriesCap": cap})
    plain = blance_b200.PlanNextMapScenarios(prev, assign, NODES, model, opts, scs, favor, wantMaps=range(len(scs)),
                                             scheduleConcurrency=counts)
    beg = dict(prev)
    beg.update({p: {} for p in assign if p not in prev})
    for sc, r, q in zip(scs, res, plain):
        assert r["next_map"] == q["next_map"] and r["schedules"] == q["schedules"] and "exposures" not in q
        final = dict(prev)
        final.update({p: r["next_map"][p] for p in assign})
        m = {s: (pri, (sc.get("modelStateConstraints") or {}).get(s, k)) for s, (pri, k) in model.items()}
        assert len(r["exposures"]) == len(counts)
        for c, e, s in zip(counts, r["exposures"], r["schedules"]):
            want = blance_b200.OrchestrateExposure(m, blance_b200.OrchestratorOptions(c, favor), NODES, beg, final, hierarchy)
            assert e["rounds"] == want["rounds"] == s["Rounds"]
            for k in want:
                if k == "kernel_ms":
                    continue
                g, w = e[k], want[k]
                if k == "series":
                    g, w = {x: list(v) for x, v in g.items()}, {x: list(v)[:cap] for x, v in w.items()}
                assert g == w, (k, c, favor)
    return res


@pytest.mark.parametrize("seed", range(3))
def test_removals_with_prev_only_partitions(seed):
    rnd = random.Random(seed)
    model = {"primary": (0, 1), "replica": (1, 2)}
    prev = prev_map(rnd, 240)
    assign = {p: v for p, v in prev.items() if rnd.random() < 0.8}          # the rest stays as in prevMap
    scs = [{"nodesToRemove": [NODES[j]], "nodesToAdd": None} for j in (0, 5)] + \
          [{"nodesToRemove": [NODES[3]], "nodesToAdd": None, "modelStateConstraints": {"primary": 1, "replica": 1}}]
    for favor in (False, True):
        check(prev, assign, model, scs, [1, 3], favor, HIERARCHY if seed else None)


def test_new_partitions_and_additions():
    rnd = random.Random(7)
    model = {"primary": (0, 1), "replica": (1, 1)}
    prev = prev_map(rnd, 150)
    assign = dict(prev)
    assign.update({"p%03d" % p: {} for p in range(150, 190)})                 # assigned, absent from prevMap
    scs = [{"nodesToRemove": [], "nodesToAdd": [NODES[11]]}, {"nodesToRemove": None, "nodesToAdd": None,
                                                              "modelStateConstraints": {"primary": 1, "replica": 2}}]
    check(prev, assign, model, scs, [2], True, HIERARCHY)


def test_series_cap_and_errors():
    rnd = random.Random(3)
    model = {"primary": (0, 1), "replica": (1, 1)}
    prev = prev_map(rnd, 120)
    scs = [{"nodesToRemove": [NODES[1]], "nodesToAdd": None}]
    full = check(prev, prev, model, scs, [1], False, None)[0]["exposures"][0]
    R = full["rounds"]
    assert R > 2
    for cap in (0, 1, R, R + 1):
        e = check(prev, prev, model, scs, [1], False, None, cap=cap)[0]["exposures"][0]
        assert all(len(v) == min(R + 1, cap) for v in e["series"].values())
        assert (e["peak"], e["area"], e["rounds"]) == (full["peak"], full["area"], R)
    with pytest.raises(blance_b200.BlanceError, match="needs scheduleConcurrency"):
        blance_b200.PlanNextMapScenarios(prev, prev, NODES, model, None, scs, exposure={})
    with pytest.raises(blance_b200.BlanceError, match="SeriesCap is negative"):
        blance_b200.PlanNextMapScenarios(prev, prev, NODES, model, None, scs, scheduleConcurrency=[1], exposure={"seriesCap": -1})
