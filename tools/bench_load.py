"""Times blance_moves_load (each node's load over the maps a rebalance passes through, on the device,
include/blance_b200.h) on the headline cluster (cfg 4: 1 048 576 partitions x 1 024 nodes, -16/+16 nodes, planned on
the GPU, with its partition weights) at MaxConcurrentPartitionMovesPerNode c = 1, 2 and 4 and both favor_min_nodes
values, against

  * the schedule call it follows (blance_moves_schedule), and
  * the host alternative: blance_moves_schedule_fetch + blance_moves_fetch and the vectorised numpy replay of
    tests/load_oracle.py, whose result is also checked against the device's.

The sweep part plans cfg 4 what-if sweeps of 8 and 66 single-node failures with schedules at c = 1, 2, 4
(blance_plan_scenarios_schedule) and the same sweeps with every (scenario, count)'s load inside the wave
(blance_plan_scenarios_load), alternating, as host clocks around the whole call, with the wave's load time and its
event-buffer bytes read from BLANCE_SCENARIO_TIMES; it reports the largest overshoot over the sweep and where.

Each arm is timed as device events (kernel_ms / device_ms) and as a host clock around the call, which ends in a
device synchronise.  Arms alternate after a warm-up of each; medians and min / max over --reps repetitions.  The
card's name, power limit and SM clocks are read in the same run.  Also reports the answer the feature exists for: the
largest overshoot of a node's load over both ends of the rebalance, the node, and the round of its peak.  Prints one
JSON object; --out also writes it to a file.

    python tools/bench_load.py [--reps 5] [--out load.json]"""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import load_oracle as LO  # noqa: E402
from bench_scenario_exposure import scenarios  # noqa: E402
from bench_scenarios import CaptureStderr, parse_waves  # noqa: E402
from bench_schedule import hardware  # noqa: E402
from blance_b200 import synth, tables  # noqa: E402


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


LOAD_RE = re.compile(r"load ([\d.]+) ms \((\d+) device bytes\)")
SWEEP_COUNTS = [1, 2, 4]


def sweep(ctx, t, scs, load):
    with CaptureStderr() as cap:                  # sets BLANCE_SCENARIO_TIMES for the call
        t0 = time.perf_counter()
        res = ctx.plan_scenarios(t, scs, False, schedule=SWEEP_COUNTS, load=load)
        s = time.perf_counter() - t0
    info = parse_waves(cap.text)
    lm = LOAD_RE.findall(cap.text)
    info.update(load_ms=round(sum(float(m[0]) for m in lm), 3), load_event_bytes=sum(int(m[1]) for m in lm))
    return res, s * 1e3, info


def sweeps(ctx, t, reps):
    out = []
    for k in (8, 66):
        scs = scenarios(t, k)
        sweep(ctx, t, scs, False)
        sweep(ctx, t, scs, True)
        ms = {"schedules": [], "schedules_and_load": []}
        for _ in range(reps):
            _, s, _ = sweep(ctx, t, scs, False)
            ms["schedules"].append(s)
            res, s, info = sweep(ctx, t, scs, True)
            ms["schedules_and_load"].append(s)
        worst = max(((r.loads[c]["over_max"], i, SWEEP_COUNTS[c], r.loads[c]["over_node"]) for i, r in enumerate(res)
                     for c in range(len(SWEEP_COUNTS))))
        out.append({"failures": k, "host_ms": {a: stats(v) for a, v in ms.items()}, "waves": info,
                    "over_max": int(worst[0]), "scenario": int(worst[1]), "c": int(worst[2]), "over_node": int(worst[3])})
        print(json.dumps(out[-1]), file=sys.stderr)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sweep-reps", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = tables.Context()
    t = synth.make_rebalance(4)
    nxt = ctx.plan_next_map(t).next_rows
    w = np.where(t.part_has_weight != 0, t.part_weight, 1).astype(np.int64)
    S = t.n_states
    res = {"hardware": hardware(), "n_parts": t.n_parts, "n_node_ids": t.n_node_ids, "reps": a.reps, "runs": []}
    for favor in (False, True):
        h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, nxt, favor, t.n_node_ids)
        for c in (1, 2, 4):
            arms = {"schedule": [], "load": []}
            dev = {"schedule": [], "load": []}
            host = []

            def schedule():
                t0 = time.perf_counter()
                _, _, sc = ctx.moves_schedule(h, c)      # its fetch is part of moves_schedule here; timed as a whole
                return time.perf_counter() - t0, sc["device_ms"], sc

            def load():
                t0 = time.perf_counter()
                r = ctx.moves_load(h, t.part_weight, t.part_has_weight)
                return time.perf_counter() - t0, r["kernel_ms"], r

            _, _, sc = schedule()
            load()
            got = None
            for _ in range(a.reps):
                s, d, sc = schedule()
                arms["schedule"].append(s * 1e3); dev["schedule"].append(d)
                s, d, got = load()
                arms["load"].append(s * 1e3); dev["load"].append(d)
            for _ in range(max(1, a.reps // 2)):
                t0 = time.perf_counter()
                ro, so, _ = ctx.moves_schedule(h, c)          # the fetch of round_off / sched_op
                off, node, state, kind = ctx.moves_fetch(h, total)
                want = LO.vectorised(t.state_slot_off, t.prev_rows, off, node, state, kind, ro, so, t.n_node_ids, w)
                host.append((time.perf_counter() - t0) * 1e3)
            LO.assert_equal(got, want, (favor, c))
            q = got["over_node"]
            res["runs"].append({
                "favor_min_nodes": favor, "c": c, "rounds": sc["rounds"], "ops": total,
                "host_ms": {k: stats(v) for k, v in arms.items()}, "device_ms": {k: stats(v) for k, v in dev.items()},
                "host_alternative_ms": stats(host),
                "over_max": int(got["over_max"]), "over_node": int(q),
                "over_node_beg": int(got["node_beg"][S][q]), "over_node_end": int(got["node_end"][S][q]),
                "over_node_peak": int(got["node_peak"][S][q]), "over_node_peak_round": int(got["node_peak_round"][S][q]),
                "nodes_over": int((got["node_peak"][S] > np.maximum(got["node_beg"][S], got["node_end"][S])).sum()),
                "max_peak": int(got["node_peak"][S].max()), "max_end": int(got["node_end"][S].max()),
            })
            print(json.dumps(res["runs"][-1]), file=sys.stderr)
        ctx.moves_free(h)
    res["sweeps"] = sweeps(ctx, t, a.sweep_reps)
    ctx.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
