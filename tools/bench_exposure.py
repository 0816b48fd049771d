"""Times blance_moves_exposure (the maps a rebalance passes through, counted per round on the device,
include/blance_b200.h) on the headline cluster (cfg 4: 1 048 576 partitions x 1 024 nodes, -16/+16 nodes, planned on
the GPU) at MaxConcurrentPartitionMovesPerNode c = 1, 2 and 4 and both favor_min_nodes values, against

  * the schedule call it follows (blance_moves_schedule), and
  * the host alternative: blance_moves_schedule_fetch + blance_moves_fetch and the vectorised numpy replay of
    tests/exposure_oracle.py, whose result is also checked against the device's.

Each arm is timed as device events (kernel_ms / device_ms) and as a host clock around the call, which ends in a
device synchronise.  Arms alternate after a warm-up of each; medians and min / max over --reps repetitions.  The
exposure with and without per-node peaks (dom_peak) is timed separately.  The card's name, power limit and SM clocks
are read in the same run.  Also reports the answer the feature exists for: the peak NO_COPY / MULTI_TOP / ONE_COPY
of every (favor_min_nodes, c).  Prints one JSON object; --out also writes it to a file.

    python tools/bench_exposure.py [--reps 5] [--out exposure.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import exposure_oracle as EO  # noqa: E402
from bench_schedule import hardware  # noqa: E402
from blance_b200 import synth, tables  # noqa: E402


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = tables.Context()
    t = synth.make_rebalance(4)
    nxt = ctx.plan_next_map(t).next_rows
    cons = np.asarray(t.state_constraints, np.int32)
    res = {"hardware": hardware(), "n_parts": t.n_parts, "n_node_ids": t.n_node_ids, "reps": a.reps, "runs": []}
    for favor in (False, True):
        h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, nxt, favor, t.n_node_ids)
        for c in (1, 2, 4):
            arms = {"schedule": [], "exposure": [], "exposure_nodom": []}
            dev = {"schedule": [], "exposure": [], "exposure_nodom": []}
            host = []
            got = None

            def schedule():
                t0 = time.perf_counter()
                _, _, sc = ctx.moves_schedule(h, c)      # its fetch is part of moves_schedule here; timed as a whole
                return time.perf_counter() - t0, sc["device_ms"], sc

            def exposure(dom=True):
                t0 = time.perf_counter()
                r = ctx.moves_exposure(h, cons, t.top_state, dom=dom)
                return time.perf_counter() - t0, r["kernel_ms"], r

            _, _, sc = schedule()
            exposure()
            exposure(dom=False)
            for _ in range(a.reps):
                s, d, sc = schedule()
                arms["schedule"].append(s * 1e3); dev["schedule"].append(d)
                s, d, got = exposure()
                arms["exposure"].append(s * 1e3); dev["exposure"].append(d)
                s, d, _ = exposure(dom=False)
                arms["exposure_nodom"].append(s * 1e3); dev["exposure_nodom"].append(d)
            for _ in range(max(1, a.reps // 2)):
                t0 = time.perf_counter()
                ro, so, _ = ctx.moves_schedule(h, c)          # the fetch of round_off / sched_op
                off, node, state, kind = ctx.moves_fetch(h, total)
                want = EO.vectorised(t.state_slot_off, t.prev_rows, off, node, state, kind, ro, so, cons, t.top_state, t.n_node_ids)
                host.append((time.perf_counter() - t0) * 1e3)
            EO.assert_equal(got, want, (favor, c))
            m = {k: i for i, k in enumerate(EO.METRICS)}
            res["runs"].append({
                "favor_min_nodes": favor, "c": c, "rounds": sc["rounds"], "ops": total,
                "host_ms": {k: stats(v) for k, v in arms.items()}, "device_ms": {k: stats(v) for k, v in dev.items()},
                "host_alternative_ms": stats(host),
                "peak": {k: int(got["peak"][i]) for k, i in m.items()},
                "peak_round": {k: int(got["peak_round"][i]) for k, i in m.items()},
                "max_dom_peak": int(got["dom_peak"].max()),
                "parts_ever_without_copy": int(((got["part_flags"] >> m["NO_COPY"]) & 1).sum()),
                "parts_ever_multi_top": int(((got["part_flags"] >> m["MULTI_TOP"]) & 1).sum()),
            })
            print(json.dumps(res["runs"][-1]), file=sys.stderr)
        ctx.moves_free(h)
    ctx.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
