"""Chains whose stages change plan options (blance_plan_chains_ex) against the one-by-one path: every stage's rows
copied out, the next stage's tables rebuilt on the host with that stage's options, one blance_plan_next_map per stage.
Prints one JSON object and writes it to --out.

    python tools/bench_chain_options.py [--ks 8,66] [--obo 2] [--out profiles/h100_chain_options.json]

Workload on cfg 4 (synth.make_rebalance(4): 1 048 576 partitions x 1 024 nodes, primary 1 + replica 2): chain j
  stage 1  removes live node j (it leaves nodesAll at stage 2);
  stage 2  raises the replica constraint from 2 to 3 (no node change);
  stage 3  adds node j back, still at 3 replicas.
The options call plans on the layout widened from 3 to 4 slots; the plain arm is the same three stages without option
changes on the 3-slot layout (blance_plan_chains), for the "device bytes each" the library prints beside it.  The
one-by-one path is measured on --obo chains and scaled to K, as tools/bench_chains.py does.  Timings are host wall
clock around calls that end in a device synchronise; the card name, power limit and clocks are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_chains import clocks, live_nodes  # noqa: E402
from bench_scenarios import gpu_info  # noqa: E402

from blance_b200 import synth, tables  # noqa: E402

REPLICA = 1            # the state index of "replica" in cfg 4


def base_tables():
    t = synth.make_rebalance(4)
    t.node_removed[:] = 0
    t.node_added[:] = 0
    t.add_is_nil = 0
    return t


def chains_of(t, nodes):
    """The three stages of each chain j, and each stage's options: [{}, raised, raised]."""
    N, NU = t.n_nodes, t.n_node_ids
    zero = np.zeros(NU, np.uint8)
    raised = np.array(t.state_constraints, np.int32)
    raised[REPLICA] += 1
    chains = []
    for j in nodes:
        rm, ad, out = zero.copy(), zero.copy(), np.ones(N, np.uint8)
        rm[j] = ad[j] = 1
        out[j] = 0
        chains.append([dict(node_removed=rm, node_added=zero, add_is_nil=0, node_in_all=np.ones(N, np.uint8)),
                       dict(node_removed=zero, node_added=zero, add_is_nil=0, node_in_all=out),
                       dict(node_removed=zero, node_added=ad, add_is_nil=0, node_in_all=np.ones(N, np.uint8))])
    return chains, [{}, dict(state_constraints=raised), dict(state_constraints=raised)]


def one_by_one(ctx, w, chain, opts):
    """One chain through blance_plan_next_map: each stage's tables built on the host from the previous stage's rows, with
    that stage's node sets, membership (the ids outside nodesAll renumbered after the members) and options."""
    import chain_util as C                       # the renumbering of tests/chain_util.py (single-plan form)
    cur, res = w, []
    for s, (stage, o) in enumerate(zip(chain, opts)):
        x = C.substituted(cur, stage, o, s)
        r, order = C.renumbered(x, stage["node_in_all"])
        out = ctx.plan_next_map(r)
        nxt = np.where(out.next_rows >= 0, order[np.maximum(out.next_rows, 0)], -1).astype(np.int32)
        res.append((nxt, out))
        cur = C.advance(cur, nxt, out.next_shape)
    return res


def scenario_log(k, widen):
    """The BLANCE_SCENARIO_TIMES lines of one call at K = k (options call when widen, else the plain chain)."""
    env = dict(os.environ, BLANCE_SCENARIO_TIMES="1")
    code = ("import sys; sys.path.insert(0, %r); import bench_chain_options as B; B.probe(%d, %r)" %
            (os.path.dirname(os.path.abspath(__file__)), k, widen))
    err = subprocess.run([sys.executable, "-c", code], env=env, stderr=subprocess.PIPE, stdout=subprocess.DEVNULL, text=True).stderr
    lines = [x for x in err.splitlines() if "[blance]" in x]
    sizes = sorted({int(x.split("wave size ")[1].split(",")[0]) for x in lines if "wave size " in x})
    each = sorted({int(x.split("device bytes each")[0].split(",")[-1]) for x in lines if "device bytes each" in x})
    return dict(wave_sizes=sizes, device_bytes_each=each, log=lines[:3])


def probe(k, widen):
    ctx = tables.Context()
    t = base_tables()
    chains, opts = chains_of(t, live_nodes(t, k))
    if widen:
        w = tables.widen_layout(t, np.asarray(opts[1]["state_constraints"]))
        ctx.plan_chains(w, chains, False, stage_opts=[opts] * k)
    else:
        ctx.plan_chains(t, chains, False)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="8,66")
    ap.add_argument("--obo", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    ctx = tables.Context()
    t = base_tables()
    rec = dict(workload="cfg 4 (1 048 576 partitions x 1 024 nodes): remove j; raise replicas 2 -> 3; add j back (T = 3)",
               **gpu_info(), **clocks(), runs=[])
    for k in [int(x) for x in a.ks.split(",")]:
        chains, opts = chains_of(t, live_nodes(t, k))
        w = tables.widen_layout(t, np.asarray(opts[1]["state_constraints"]))
        ctx.plan_chains(w, chains[:1], False, stage_opts=[opts])                  # warm-up
        t0 = time.perf_counter()
        res, nets = ctx.plan_chains(w, chains, False, stage_opts=[opts] * k, want_rows=[(i, s) for i in range(a.obo) for s in range(3)])
        ex_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        ctx.plan_chains(t, chains, False)
        plain_s = time.perf_counter() - t0
        n_one = min(k, a.obo)
        t0 = time.perf_counter()
        ones = [one_by_one(ctx, w, chains[i], opts) for i in range(n_one)]
        one_s = (time.perf_counter() - t0) / n_one * k
        for i, stages in enumerate(ones):
            for s, (nxt, r) in enumerate(stages):
                got = res[i][s]
                assert np.array_equal(got.next_rows, nxt) and np.array_equal(got.warn, r.warn), (k, i, s)
                assert (got.iters_run, got.converged, got.steps) == (r.iters_run, r.converged, r.steps), (k, i, s)
        run = dict(K=k, chains_ex_s=round(ex_s, 3), plain_chain_s=round(plain_s, 3), one_by_one_s=round(one_s, 3),
                   one_by_one_measured_chains=n_one, speedup_vs_one_by_one=round(one_s / ex_s, 2), sampled_stages_equal=3 * n_one,
                   ops_total_mean=[float(np.mean([res[i][s].ops_total for i in range(k)])) for s in range(3)],
                   net_ops_total_mean=float(np.mean([n.ops_total for n in nets])),
                   iters=[[res[i][s].iters_run for s in range(3)] for i in range(min(k, 2))],
                   options_call=scenario_log(k, True), plain_chain=scenario_log(k, False))
        rec["runs"].append(run)
        print(json.dumps(run), flush=True)
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
