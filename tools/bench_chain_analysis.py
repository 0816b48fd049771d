"""Schedules, audits and exposures of every chain stage through blance_plan_chains_exposure, against the plain chain call
and against the one-by-one path (each stage's rows copied out, then blance_moves_create / _schedule / _exposure per
count and blance_map_audit), alternating arms in one process, medians.  Prints one JSON object and writes it to --out.

    python tools/bench_chain_analysis.py [--ks 8,66] [--reps 3] [--out profiles/h100_chain_analysis.json]

Workload: the cfg 4 rolling upgrade of tools/bench_chains.py (1 M partitions x 1 024 nodes; chain j removes live node j,
then adds it back: T = 2), counts c = 1, 2, 4, both favor_min_nodes.  Arms:
  plain      blance_plan_chains
  sched      + schedules (per-stage summaries)
  full       + audits and exposures (per-stage per-partition arrays, dom peaks), and full_nodom without dom
  span       the span only: no per-stage array
  one_by_one measured on --obo chains and scaled to K: rows out, then the handle path per stage and count
Then one long chain (--long-T stages on cfg 4, 4 chains, rebalances with no node change after the first removal): the
span alone against every per-stage array copied out.  Timings are host wall clock around calls that end in a device
synchronise; the wave size is read from BLANCE_SCENARIO_TIMES' log of one extra call."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_chains import clocks, live_nodes, rolling  # noqa: E402
from bench_scenarios import gpu_info  # noqa: E402

from blance_b200 import synth, tables  # noqa: E402

COUNTS = [1, 2, 4]


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def arms(ctx, t, chains, favor):
    full = dict(schedule=COUNTS, audit={}, exposure=dict(series_cap=64), span=True)
    return {
        "plain": lambda: ctx.plan_chains(t, chains, favor),
        "sched": lambda: ctx.plan_chains(t, chains, favor, schedule=COUNTS),
        "full": lambda: ctx.plan_chains(t, chains, favor, **full),
        "full_nodom": lambda: ctx.plan_chains(t, chains, favor, schedule=COUNTS, audit={}, exposure=dict(series_cap=64, dom=False), span=True),
        "span": lambda: ctx.plan_chains(t, chains, favor, schedule=COUNTS, exposure=dict(), span=True, stage_arrays=False),
    }


def one_by_one(ctx, t, chains, favor):
    """The chains planned with their rows out, then every stage analysed through the handle path."""
    T = len(chains[0])
    res, _ = ctx.plan_chains(t, chains, favor, want_rows=[(i, s) for i in range(len(chains)) for s in range(T)])
    mover = (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8)
    cons = np.asarray(t.state_constraints, np.int32)
    for i in range(len(chains)):
        cur_rows, in_prev = np.asarray(t.prev_rows).reshape(t.n_parts, -1), np.asarray(t.part_in_prev) != 0
        assigned = np.asarray(t.part_in_assign) != 0
        for s in range(T):
            r = res[i][s]
            member = in_prev | assigned
            beg = np.where(in_prev[:, None], cur_rows, -1).astype(np.int32)
            end = np.where(assigned[:, None], r.next_rows, beg).astype(np.int32)
            h, _ = ctx.moves_create(t.state_slot_off, beg[member], end[member], favor, t.n_node_ids)
            for c in COUNTS:
                ctx.moves_schedule(h, c, mover)
                ctx.moves_exposure(h, cons, t.top_state, None)
            ctx.moves_free(h)
            ctx.map_audit(t, end, np.where(assigned[:, None], r.next_shape, t.prev_shape.reshape(t.n_parts, -1)))
            cur_rows, in_prev = end, member


def wave_size(args):
    """The wave size the automatic sizing picks for the full arm at K = args[0], read from BLANCE_SCENARIO_TIMES."""
    env = dict(os.environ, BLANCE_SCENARIO_TIMES="1")
    code = ("import sys; sys.path.insert(0, %r); import bench_chain_analysis as B; B.probe(%d)" %
            (os.path.dirname(os.path.abspath(__file__)), args))
    err = subprocess.run([sys.executable, "-c", code], env=env, stderr=subprocess.PIPE, stdout=subprocess.DEVNULL, text=True).stderr
    sizes = sorted({int(x.split("wave size ")[1].split(",")[0]) for x in err.splitlines() if "wave size " in x})
    return sizes, [x for x in err.splitlines() if "[blance]" in x][:4]


def probe(k):
    ctx = tables.Context()
    t = synth.make_rebalance(4)
    ctx.plan_chains(t, rolling(t, live_nodes(t, k)), False, schedule=COUNTS, audit={}, exposure=dict(series_cap=64), span=True)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--obo", type=int, default=2)
    ap.add_argument("--long-T", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = tables.Context()
    t = synth.make_rebalance(4)
    out = dict(workload="cfg4 rolling upgrade, 1048576 partitions x 1024 nodes, T = 2, counts %s" % COUNTS, gpu=gpu_info(), clocks=clocks(),
               timing="host wall clock around calls that end in a device synchronise; medians over --reps alternated rounds", runs=[])
    for k in [int(x) for x in a.ks.split(",")]:
        chains = rolling(t, live_nodes(t, k))
        for favor in (False, True):
            fs = arms(ctx, t, chains, favor)
            for f in fs.values():                    # warm-up of every shape
                f()
            ms = {name: [] for name in fs}
            ms["one_by_one_sample"] = []
            for _ in range(a.reps):
                for name, f in fs.items():
                    ms[name].append(timed(f)[0])
                ms["one_by_one_sample"].append(timed(lambda: one_by_one(ctx, t, chains[:a.obo], favor))[0])
            med = {name: float(np.median(v)) for name, v in ms.items()}
            med["one_by_one_scaled_to_K"] = med.pop("one_by_one_sample") * k / a.obo
            out["runs"].append(dict(K=k, favor_min_nodes=favor, ms=med))
        sizes, log = wave_size(k)
        out["runs"][-1]["wave_sizes_full_arm"] = sizes
        out["runs"][-1]["scenario_times_log"] = log
    # one long chain: the first stage removes a node, then rebalances with no node change
    T = a.long_T
    nodes = live_nodes(t, 4)
    chains = []
    for c in rolling(t, nodes):
        rest = [dict(c[1], node_added=np.zeros(t.n_node_ids, np.uint8)) for _ in range(T - 1)]
        rest[-1] = c[1]
        chains.append([c[0]] + rest)
    long_arms = {
        "span_only": lambda: ctx.plan_chains(t, chains, False, schedule=COUNTS, exposure=dict(), span=True, stage_arrays=False),
        "per_stage_arrays": lambda: ctx.plan_chains(t, chains, False, schedule=COUNTS, exposure=dict(series_cap=64), span=True),
    }
    for f in long_arms.values():
        f()
    lm = {name: [] for name in long_arms}
    for _ in range(max(1, a.reps - 1)):
        for name, f in long_arms.items():
            lm[name].append(timed(f)[0])
    P, NU = t.n_parts, t.n_node_ids
    out["long_chain"] = dict(chains=4, T=T, ms={k: float(np.median(v)) for k, v in lm.items()},
                             per_stage_host_bytes=int(4 * len(COUNTS) * (P * (4 + 4 + 4 + 1) + NU * 8 + NU * (8 + 4))),
                             note="per_stage_host_bytes: the per-partition and per-node arrays of 4 chains x counts per stage "
                                  "(part_done, part_min_copies, part_no_top, part_flags; node_rounds, node_last; dom peak, round)")
    ctx.close()
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
