"""What-if branches off the stages of a rolling upgrade (blance_plan_chain_branches) against the path without forks:
one blance_plan_chains_ex call per branch point on the branches' equivalent chains, each replanning the trunk prefix.
Prints one JSON object and writes it to --out.

    python tools/bench_chain_branches.py [--k 4] [--f 4] [--out profiles/h100_chain_branches.json]

Workload on cfg 4 (synth.make_rebalance(4): 1 048 576 partitions x 1 024 nodes, primary 1 + replica 2): K trunk
chains of T = 3 stages, a rolling upgrade of two nodes a_j, b_j per chain j:
  stage 0  takes a_j out;
  stage 1  brings a_j back and takes b_j out;
  stage 2  brings b_j back.
After every trunk stage t of every chain, F branches of one stage each: "node x fails now" for F live nodes x.  The
branch call plans K.T + K.F.T stages; the baseline plans the trunk (K.T) and, per branch point t, the K.F equivalent
chains of t + 2 stages.  Every branch's summaries and loop counters are checked against its equivalent chain's last
stage.  Timings are host wall clock around calls that end in a device synchronise; the card name, power limit and clocks
are read in the same run, and the library's BLANCE_SCENARIO_TIMES lines give the device bytes of each wave member."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_chains import clocks  # noqa: E402
from bench_scenarios import gpu_info  # noqa: E402

from blance_b200 import synth, tables  # noqa: E402

T = 3


def base_tables():
    t = synth.make_rebalance(4)
    t.node_removed[:] = 0
    t.node_added[:] = 0
    t.add_is_nil = 0
    return t


def workload(t, k, f):
    """The K trunk chains and the branches (one stage each) after every stage."""
    N, NU = t.n_nodes, t.n_node_ids
    live = [q for q in range(N)]
    zero = np.zeros(NU, np.uint8)

    def stage(rm=(), ad=(), out=()):
        r, a, m = zero.copy(), zero.copy(), np.ones(N, np.uint8)
        r[list(rm)] = 1
        a[list(ad)] = 1
        m[list(out)] = 0
        return dict(node_removed=r, node_added=a, add_is_nil=0, node_in_all=m)

    chains, branches = [], []
    for j in range(k):
        a, b = live[2 * j], live[2 * j + 1]
        chains.append([stage(rm=[a]), stage(rm=[b], ad=[a], out=[a]), stage(ad=[b], out=[b])])
        out_after = [[a], [b], []]                   # outside nodesAll at the stage after trunk stage t
        for s in range(T):
            fails = [q for q in live[2 * k:] if q not in (a, b)][(j * T + s) * f:(j * T + s + 1) * f]
            for x in fails:
                branches.append(dict(chain=j, after_stage=s, stages=[stage(rm=[x], out=out_after[s])], stage_opts=None))
    return chains, branches


def scenario_log(k, f):
    """The BLANCE_SCENARIO_TIMES lines of one branch call."""
    env = dict(os.environ, BLANCE_SCENARIO_TIMES="1")
    code = ("import sys; sys.path.insert(0, %r); import bench_chain_branches as B; B.probe(%d, %d)" %
            (os.path.dirname(os.path.abspath(__file__)), k, f))
    err = subprocess.run([sys.executable, "-c", code], env=env, stderr=subprocess.PIPE, stdout=subprocess.DEVNULL, text=True).stderr
    lines = [x for x in err.splitlines() if "[blance]" in x]
    trunk = [x for x in lines if "branches after" not in x]
    branch = [x for x in lines if "branches after" in x]
    each = lambda ls: sorted({int(x.split("device bytes each")[0].split(",")[-1]) for x in ls if "device bytes each" in x})  # noqa: E731
    sizes = lambda ls: sorted({int(x.split("wave size ")[1].split(",")[0]) for x in ls if "wave size " in x})  # noqa: E731
    return dict(trunk_wave_sizes=sizes(trunk), trunk_device_bytes_each=each(trunk), branch_wave_sizes=sizes(branch),
                branch_device_bytes_each=each(branch), trunk_log=trunk[:T], branch_log=branch[:T])


def probe(k, f):
    ctx = tables.Context()
    t = base_tables()
    chains, branches = workload(t, k, f)
    ctx.plan_chains(t, chains, False, stage_opts=[[{}] * T] * k, branches=branches)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--f", type=int, default=4)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    k, f = a.k, a.f
    ctx = tables.Context()
    t = base_tables()
    chains, branches = workload(t, k, f)
    so = [[{}] * T] * k
    rec = dict(workload="cfg 4 (1 048 576 partitions x 1 024 nodes): K = %d rolling upgrades of T = %d stages, F = %d one-stage "
                        "node-failure branches after every stage" % (k, T, f), **gpu_info(), **clocks(), runs=[])
    rec["stage_plans"] = dict(branch_call=k * T + k * f * T, chains_ex_per_point=k * T + sum(k * f * (s + 2) for s in range(T)))
    ctx.plan_chains(t, chains[:1], False, stage_opts=so[:1], branches=branches[:1])         # warm-up
    for rep in range(a.repeat):
        t0 = time.perf_counter()
        res, nets, bres, bnets = ctx.plan_chains(t, chains, False, stage_opts=so, branches=branches)
        br_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        tres, tnets = ctx.plan_chains(t, chains, False, stage_opts=so)
        eq = {}
        for s in range(T):
            idx = [b for b, x in enumerate(branches) if x["after_stage"] == s]
            eqc = [chains[branches[b]["chain"]][:s + 1] + branches[b]["stages"] for b in idx]
            r, n = ctx.plan_chains(t, eqc, False, stage_opts=[[{}] * (s + 2)] * len(eqc))
            for x, b in enumerate(idx):
                eq[b] = (r[x][s + 1], n[x])
        base_s = time.perf_counter() - t0
        checked = 0
        for b in range(len(branches)):
            got, want = bres[b][0], eq[b][0]
            for fld in ("iters_run", "converged", "steps", "parts_moved", "ops_total", "warn_parts"):
                assert getattr(got, fld) == getattr(want, fld), (b, fld)
            assert np.array_equal(got.node_ops, want.node_ops) and np.array_equal(got.state_node_load, want.state_node_load), b
            assert bnets[b].ops_total == eq[b][1].ops_total and np.array_equal(bnets[b].node_ops, eq[b][1].node_ops), b
            checked += 1
        for i in range(k):
            for s in range(T):
                assert res[i][s].ops_total == tres[i][s].ops_total and np.array_equal(res[i][s].node_ops, tres[i][s].node_ops)
        run = dict(repeat=rep, branch_call_s=round(br_s, 3), chains_ex_per_point_s=round(base_s, 3), speedup=round(base_s / br_s, 2),
                   branches_checked=checked, branch_ops_total_mean=float(np.mean([r[0].ops_total for r in bres])))
        rec["runs"].append(run)
        print(json.dumps(run), flush=True)
    ctx.close()
    rec["scenario_log"] = scenario_log(k, f)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
