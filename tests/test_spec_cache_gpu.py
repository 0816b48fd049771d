"""The speculative pass kernel's cached base keys and its extended resolve (assign_pass_spec.cuh).

When the leader's bound proof fails with K winners, the leader scans the cached base keys for the nodes between ub
and the K-th winner and scores them itself; when there are more than SP_XMAX of them the team evaluates the step.
Every case here plans with the speculative kernel (auto engine, no sequencer) against the array-form CPU oracle on
the same tables, bit for bit, and reads the kernel's path counters (BLANCE_SPEC_STATS) to show which paths ran:
reduced cfg-4 clusters with the replica constraint at 1-4 and 768 / 1 024 / 2 048 nodes, and clusters whose node
weights are nearly all equal, so that the tie groups of equal base keys are large and the extended set is sometimes
larger than SP_XMAX.  Needs an H100; run with `-m gpu`."""
import re

import numpy as np
import pytest

from test_engine_limits_gpu import SPEC, assert_kernel, assert_same, cluster, oracle_tables, set_engine

from blance_b200 import synth, tables

pytestmark = pytest.mark.gpu

STATS = re.compile(r"team: full after a failed proof (\d+) .*\| full, other rows (\d+) .*\| rebuild, list dry (\d+) .*"
                   r"\| full that moved (\d+) .*\| extended resolves (\d+), too large (\d+)")
FIELDS = ("full_proof", "full_other", "rebuild_dry", "full_moved", "xres", "xover")


@pytest.fixture(scope="module")
def ctx():
    c = tables.Context()
    yield c
    c.close()


def plan_counted(ctx, monkeypatch, capfd, t, what):
    """Plans t with the speculative kernel, checks it against the oracle and returns the kernel's path counters."""
    ref = oracle_tables(t)
    set_engine(monkeypatch, t, SPEC)
    monkeypatch.setenv("BLANCE_SPEC_STATS", "1")
    capfd.readouterr()
    got = ctx.plan_next_map(t)
    err = capfd.readouterr().err
    assert_same(got, ref, what)
    assert_kernel(got, SPEC, what)
    lines = [m for m in (STATS.search(l) for l in err.splitlines()) if m]
    assert lines, (what, err[-2000:])
    counts = dict(zip(FIELDS, (sum(int(m.group(i + 1)) for m in lines) for i in range(len(FIELDS)))))
    with capfd.disabled():
        print(what, counts)
    return counts


def cfg4(N, K, P=16384):
    """The cfg-4 rebalance at N nodes with the replica constraint at K (slots widened where K > 2)."""
    t = synth.make_rebalance(4, P=P, N=N)
    if K > 2:
        t = tables.widen_layout(t, [1, K])
    return tables.scenario_tables(t, {}, dict(state_constraints=np.array([1, K], np.int32)))


def equal_weights(N, K, P=8192, seed=0, frac=0.95):
    """cluster() with almost every node of weight 1: large groups of nodes share one base key."""
    t = cluster(N, P, [1, K], n_rm=4, n_add=4, seed=seed)
    rng = np.random.default_rng(seed + 100)
    t.node_weight[:] = np.where(rng.random(N) < frac, 1, rng.integers(2, 5, N)).astype(t.node_weight.dtype)
    return t


@pytest.mark.parametrize("N", [768, 1024, 2048])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_cfg4_every_constraint_and_node_count(ctx, monkeypatch, capfd, N, K):
    plan_counted(ctx, monkeypatch, capfd, cfg4(N, K), ("cfg4", N, K))


@pytest.mark.parametrize("N", [768, 1024, 2048])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_equal_weights_every_constraint_and_node_count(ctx, monkeypatch, capfd, N, K):
    plan_counted(ctx, monkeypatch, capfd, equal_weights(N, K, seed=K), ("equal weights", N, K))


def test_leader_local_and_team_paths_both_run(ctx, monkeypatch, capfd):
    """On these clusters failed proofs are resolved by the leader AND handed to the team when the extended set is too
    large; both give the oracle's result."""
    total = dict.fromkeys(FIELDS, 0)
    for what, t in (("cfg4 1024 x 65536", cfg4(1024, 2, P=65536)), ("equal weights 1024", equal_weights(1024, 2, P=16384))):
        c = plan_counted(ctx, monkeypatch, capfd, t, what)
        total = {k: total[k] + c[k] for k in FIELDS}
    assert total["xres"] > 0, total
    assert total["xover"] > 0, total
    assert total["full_proof"] >= total["xover"], total
