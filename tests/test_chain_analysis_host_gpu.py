"""blance_b200.PlanNextMapChains(..., scheduleConcurrency, audit, exposure) over string maps: every stage's exposure at
every count equals OrchestrateExposure on that stage's begMap (the stage's prevMap plus an empty entry for every
assigned partition it lacks) and final map, every stage's audit equals AuditMap of its final map, the net rebalance
equals OrchestrateExposure from prevMap to the last stage's map, and the span folds the stages.  Names are
fixed-width, so interning order equals byte order.  Needs an H100; run with -m gpu."""
import random

import pytest

import blance_b200
from test_scenario_exposure_host_gpu import HIERARCHY, NODES, prev_map

pytestmark = pytest.mark.gpu
CAP = 4096


def same_exposure(got, want, what):
    assert got["rounds"] == want["rounds"], what
    for k in want:
        if k == "kernel_ms":
            continue
        g, w = got[k], want[k]
        if k == "series":
            g, w = {x: list(v) for x, v in g.items()}, {x: list(v)[:CAP] for x, v in w.items()}
        assert g == w, (what, k)


@pytest.mark.parametrize("favor", [False, True])
def test_rolling_upgrade_matches_orchestrate_exposure_and_audit_map(favor):
    rnd = random.Random(5 + favor)
    model = {"primary": (0, 1), "replica": (1, 2)}
    prev = prev_map(rnd, 200)
    assign = {p: v for p, v in prev.items() if rnd.random() < 0.85}          # the rest stays as in prevMap
    chains = [{"stages": [{"nodesToRemove": [q], "nodesToAdd": None}, {"nodesToRemove": None, "nodesToAdd": [q]}]}
              for q in (NODES[2], NODES[7])]
    chains.append({"modelStateConstraints": {"primary": 1, "replica": 1},
                   "stages": [{"nodesToRemove": [NODES[0]], "nodesToAdd": None}, {"nodesToRemove": [NODES[4]], "nodesToAdd": None}]})
    counts = [1, 3]
    opts = blance_b200.PlanNextMapOptions(NodeHierarchy=HIERARCHY)
    res = blance_b200.PlanNextMapChains(prev, assign, NODES, model, opts, chains, favor, wantMaps=range(len(chains)),
                                        scheduleConcurrency=counts, audit={}, exposure={"seriesCap": CAP})
    plain = blance_b200.PlanNextMapChains(prev, assign, NODES, model, opts, chains, favor, wantMaps=range(len(chains)))
    for i, (chain, r, q) in enumerate(zip(chains, res, plain)):
        m = {s: (pri, (chain.get("modelStateConstraints") or {}).get(s, k)) for s, (pri, k) in model.items()}
        aopts = blance_b200.PlanNextMapOptions(NodeHierarchy=HIERARCHY, ModelStateConstraints=chain.get("modelStateConstraints"))
        assert r["net"]["node_ops"] == q["net"]["node_ops"]
        cur = dict(prev)
        for t, (s, sq) in enumerate(zip(r["stages"], q["stages"])):
            assert s["next_map"] == sq["next_map"] and s["node_ops"] == sq["node_ops"]
            beg = dict(cur)
            beg.update({p: {} for p in assign if p not in cur})
            final = dict(cur)
            final.update({p: s["next_map"][p] for p in assign})
            assert s["audit"] == blance_b200.AuditMap(final, NODES, model, aopts), (i, t)
            for c, e, sch in zip(counts, s["exposures"], s["schedules"]):
                want = blance_b200.OrchestrateExposure(m, blance_b200.OrchestratorOptions(c, favor), NODES, beg, final, HIERARCHY)
                same_exposure(e, want, (i, t, c))
                assert sch["Rounds"] == want["rounds"]
            cur = final
        beg0 = dict(prev)
        beg0.update({p: {} for p in assign if p not in prev})
        for k, c in enumerate(counts):
            want = blance_b200.OrchestrateExposure(m, blance_b200.OrchestratorOptions(c, favor), NODES, beg0, cur, HIERARCHY)
            same_exposure(r["net"]["exposures"][k], want, (i, "net", c))
            assert r["net"]["schedules"][k]["Rounds"] == want["rounds"]
            sp = r["span"][k]
            stages = [s["exposures"][k] for s in r["stages"]]
            assert sp["rounds"] == sum(s["schedules"][k]["Rounds"] for s in r["stages"])
            assert sp["moves_done"] == sum(s["schedules"][k]["MovesDone"] for s in r["stages"])
            for metric in sp["peak"]:
                assert sp["peak"][metric] == max(e["peak"][metric] for e in stages)
                assert sp["area"][metric] == sum(e["area"][metric] for e in stages)
            for name, v in sp["dom_peak"].items():
                assert v == max(e["dom_peak"].get(name, 0) for e in stages)
            for node, v in sp["node_rounds"].items():
                assert v == sum(s["schedules"][k]["NodeRounds"].get(node, 0) for s in r["stages"])


def test_errors():
    rnd = random.Random(3)
    model = {"primary": (0, 1), "replica": (1, 1)}
    prev = prev_map(rnd, 40)
    chains = [{"stages": [{"nodesToRemove": [NODES[1]], "nodesToAdd": None}]}]
    with pytest.raises(blance_b200.BlanceError, match="needs scheduleConcurrency"):
        blance_b200.PlanNextMapChains(prev, prev, NODES, model, None, chains, exposure={})
    with pytest.raises(blance_b200.BlanceError, match="SeriesCap is negative"):
        blance_b200.PlanNextMapChains(prev, prev, NODES, model, None, chains, scheduleConcurrency=[1], exposure={"seriesCap": -1})
