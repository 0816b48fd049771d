"""blance_b200.OrchestrateLoad over string maps: equal to a literal replay of OrchestrateSchedule's batches, as the
reference's test app applies AssignPartitionsFunc calls (orchestrate_test.go:137-157), with and without partition
weights.  Needs an H100; run with -m gpu."""
import random

import pytest

import blance_b200
from test_exposure_host_gpu import random_maps

pytestmark = pytest.mark.gpu


def replay(begMap, rounds, weights):
    """Each node's load over the maps `rounds` (OrchestrateSchedule's batches) pass through, keyed as OrchestrateLoad
    keys it."""
    maps = {p: [(n, s) for s, lst in nbs.items() for n in (lst or [])] for p, nbs in begMap.items()}
    w = {p: (weights or {}).get(p, 1) for p in maps}
    series = []                                      # per t: {(state or None, node): load}
    for t in range(len(rounds) + 1):
        if t:
            for call in rounds[t - 1]:
                for p, s in zip(call.Partitions, call.States):
                    maps[p] = [e for e in maps[p] if e[0] != call.Node] + ([(call.Node, s)] if s else [])
        load = {}
        for p, ents in maps.items():
            for n, s in ents:
                for k in ((s, n), (None, n)):
                    load[k] = load.get(k, 0) + w[p]
        series.append(load)
    keys = {k for d in series for k in d}
    states, nodes = {}, {}
    for k in keys:
        v = [d.get(k, 0) for d in series]
        if max(v) == 0:
            continue
        one = dict(beg=v[0], end=v[-1], peak=max(v), peak_round=v.index(max(v)))
        if k[0] is None:
            nodes[k[1]] = one
        else:
            states.setdefault(k[0], {})[k[1]] = one
    over = {n: l["peak"] - max(l["beg"], l["end"]) for n, l in nodes.items()}
    return dict(rounds=len(rounds), states=states, nodes=nodes, over_max=max(over.values(), default=0), over=over)


def check(model, nodesAll, beg, end, conc, favor, weights=None):
    opts = blance_b200.OrchestratorOptions(MaxConcurrentPartitionMovesPerNode=conc, FavorMinNodes=favor)
    got = blance_b200.OrchestrateLoad(model, opts, nodesAll, beg, end, weights)
    rounds = blance_b200.OrchestrateSchedule(model, opts, nodesAll, beg, end)
    want = replay(beg, rounds, weights)
    for k in ("rounds", "states", "nodes", "over_max"):
        assert got[k] == want[k], (k, conc, favor)
    assert want["over"].get(got["over_node"], 0) == got["over_max"]
    return got


def test_primary_swap_overshoots_both_nodes():
    model = {"primary": (0, 1), "replica": (1, 1)}
    beg = {"p": {"primary": ["a"]}, "q": {"primary": ["b"]}}
    end = {"p": {"primary": ["b"]}, "q": {"primary": ["a"]}}
    two = check(model, ["a", "b"], beg, end, 1, False, {"p": 3, "q": 3})
    assert two["over_max"] == 3 and two["over_node"] == "a"
    assert two["nodes"]["a"] == dict(beg=3, end=3, peak=6, peak_round=1)
    one = check(model, ["a", "b"], beg, end, 1, True, {"p": 3, "q": 3})
    assert one["over_max"] == 0 and one["nodes"]["b"] == dict(beg=3, end=3, peak=3, peak_round=0)


@pytest.mark.parametrize("seed", range(6))
def test_random_string_maps_equal_the_replay(seed):
    rnd = random.Random(100 + seed)
    nodes = ["n%d" % i for i in range(7)]
    model = {"primary": (0, 1), "replica": (1, 2)} if seed % 2 else {"primary": (0, 1), "replica": (1, 1), "zz": (0, 0)}
    beg, end = random_maps(rnd, nodes, sorted(model), 40)
    nodesAll = nodes if seed % 3 else nodes[:-1]          # the last node without a mover: stuck partitions
    weights = None if seed < 3 else {p: rnd.randint(0, 9) for p in rnd.sample(sorted(beg), 25)}
    for conc in (1, 2, 4):
        for favor in (False, True):
            check(model, nodesAll, beg, end, conc, favor, weights)


def test_bad_weight_and_mismatched_maps():
    m = {"0": {"primary": ["a"]}}
    with pytest.raises(blance_b200.BlanceError, match="outside \\[0, 999999999\\]"):
        blance_b200.OrchestrateLoad({"primary": (0, 1)}, None, ["a"], m, m, {"0": -1})
    with pytest.raises(blance_b200.BlanceError, match="mismatched begMap and endMap"):
        blance_b200.OrchestrateLoad({"primary": (0, 1)}, None, ["a"], m, {})
