"""Chains of cluster changes through blance_plan_chains against the same stages planned one by one with
blance_plan_next_map (rows copied out, the next stage's tables rebuilt on the host), alternating in one process, with
sampled stages checked equal.  Prints one JSON object and writes it to --out.

    python tools/bench_chains.py [--ks 8,66] [--out profiles/h100_chains.json]

Rolling upgrade on cfg 4 (synth.make_rebalance(4): 1 M partitions x 1 024 nodes): chain j takes live node j out
(stage 1: nodesToRemove = [j] on top of nothing else) and puts it back (stage 2: nodesToAdd = [j]).  K chains go in
one call; the one-by-one path plans 2 K instances, each stage's tables built from the previous stage's rows by the
chain rule of include/blance_b200.h.  Then a T = 3 chain on the headline map: its own removals and additions, then
two rebalances with no node change (the removed nodes outside nodesAll).  Timings are host wall clock around calls
that end in a device synchronise."""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_scenarios import gpu_info  # noqa: E402

from blance_b200 import synth, tables  # noqa: E402


def clocks():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        sm, sm_max, mem = [x.strip() for x in out.splitlines()[0].split(",")]
        return dict(sm_clock=sm, sm_clock_max=sm_max, mem_clock=mem)
    except Exception as e:   # noqa: BLE001 - recorded, not fatal
        return dict(clocks="unknown (%s)" % e)


def advance(t, res):
    """The chain rule on flat tables: the next stage's partition tables from a stage's next rows and shapes."""
    a = t.part_in_assign != 0
    c = copy.copy(t)
    c.prev_rows = np.where(a[:, None], res.next_rows, t.prev_rows).astype(np.int32)
    c.cur_rows = np.where(a[:, None], res.next_rows, t.cur_rows).astype(np.int32)
    c.prev_shape = np.where(a[:, None], res.next_shape, t.prev_shape).astype(np.uint8)
    c.cur_shape = np.where(a[:, None], res.next_shape, t.cur_shape).astype(np.uint8)
    c.part_in_prev = np.where(a, 1, t.part_in_prev).astype(np.uint8)
    c.extra_tot_first = np.array(t.extra_tot_rest, np.int32)
    return c


def live_nodes(t, k):
    return [q for q in range(t.n_nodes) if not t.node_removed[q] and not t.node_added[q]][:k]


def rolling(t, nodes):
    N, NU = t.n_nodes, t.n_node_ids
    zero = np.zeros(NU, np.uint8)
    chains = []
    for j in nodes:
        rm, ad = zero.copy(), zero.copy()
        rm[j] = ad[j] = 1
        chains.append([dict(node_removed=rm, node_added=zero, add_is_nil=0, node_in_all=np.ones(N, np.uint8)),
                       dict(node_removed=zero, node_added=ad, add_is_nil=0, node_in_all=np.ones(N, np.uint8))])
    return chains


def one_by_one(ctx, base, j):
    """Stage 1 and 2 of chain j through blance_plan_next_map, the rows out and the tables rebuilt in between."""
    t1 = copy.copy(base)
    t1.node_removed = np.zeros(base.n_node_ids, np.uint8)
    t1.node_removed[j] = 1
    t1.node_added = np.zeros(base.n_node_ids, np.uint8)
    t1.add_is_nil = 0
    r1 = ctx.plan_next_map(t1)
    t2 = advance(t1, r1)
    t2.node_removed = np.zeros(base.n_node_ids, np.uint8)
    t2.node_added = np.zeros(base.n_node_ids, np.uint8)
    t2.node_added[j] = 1
    r2 = ctx.plan_next_map(t2)
    return r1, r2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="8,66")
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = tables.Context()
    base = synth.make_rebalance(4)
    base.node_removed[:] = 0
    base.node_added[:] = 0
    rec = dict(workload="cfg 4 (1 048 576 partitions x 1 024 nodes), rolling upgrade: remove j, then add j back",
               **gpu_info(), **clocks(), rolling=[])
    for k in [int(x) for x in args.ks.split(",")]:
        nodes = live_nodes(base, k)
        chains = rolling(base, nodes)
        ctx.plan_chains(base, chains[:1], False)                        # warm-up
        t0 = time.perf_counter()
        res, nets = ctx.plan_chains(base, chains, False, want_rows=[(i, s) for i in range(args.samples) for s in range(2)])
        chain_s = time.perf_counter() - t0
        n_one = min(k, args.samples)
        t0 = time.perf_counter()
        ones = [one_by_one(ctx, base, j) for j in nodes[:n_one]]
        one_s = (time.perf_counter() - t0) / n_one * k
        for i, (r1, r2) in enumerate(ones):
            for s, r in enumerate((r1, r2)):
                got = res[i][s]
                assert np.array_equal(got.next_rows, r.next_rows) and np.array_equal(got.warn, r.warn), (k, i, s)
                assert (got.iters_run, got.converged, got.steps) == (r.iters_run, r.converged, r.steps), (k, i, s)
        ops = [[res[i][s].ops_total for s in range(2)] for i in range(k)]
        rec["rolling"].append(dict(
            K=k, chain_call_s=round(chain_s, 3), one_by_one_s=round(one_s, 3), one_by_one_measured_chains=n_one,
            speedup=round(one_s / chain_s, 2), sampled_stages_equal=2 * n_one,
            ops_total_stage1_mean=float(np.mean([o[0] for o in ops])), ops_total_stage2_mean=float(np.mean([o[1] for o in ops])),
            net_ops_total_mean=float(np.mean([n.ops_total for n in nets])),
            back_to_start=int(sum(n.ops_total == 0 for n in nets)),
            iters=[[res[i][s].iters_run for s in range(2)] for i in range(min(k, 4))]))
        print(json.dumps(rec["rolling"][-1]), flush=True)
    # T = 3 on the headline map: its own removals / additions, then two rebalances without node changes
    head = synth.make_rebalance(4)
    N = head.n_nodes
    members = (head.node_removed[:N] == 0).astype(np.uint8)
    zero = np.zeros(head.n_node_ids, np.uint8)
    chain = [dict(node_removed=head.node_removed.copy(), node_added=head.node_added.copy(), add_is_nil=int(head.add_is_nil),
                  node_in_all=np.ones(N, np.uint8))] + [dict(node_removed=zero, node_added=zero, add_is_nil=0, node_in_all=members)] * 2
    ctx.plan_chains(head, [chain], False)
    t0 = time.perf_counter()
    res, nets = ctx.plan_chains(head, [chain], False)
    t3 = time.perf_counter() - t0
    t0 = time.perf_counter()
    ctx.plan_chains(head, [chain[:1]], False)
    t1 = time.perf_counter() - t0
    rec["no_change_T3"] = dict(call_s=round(t3, 3), one_stage_call_s=round(t1, 3),
                               stages=[dict(iters_run=r.iters_run, converged=r.converged, ops_total=r.ops_total,
                                            parts_moved=r.parts_moved, steps=r.steps) for r in res[0]],
                               net_ops_total=nets[0].ops_total)
    print(json.dumps(rec["no_change_T3"]), flush=True)
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
