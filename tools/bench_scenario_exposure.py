"""The exposure of every scenario's rebalance inside the scenario wave (blance_plan_scenarios_exposure) against the
sweep without it and against the one-by-one path, on cfg 4.  Prints JSON lines and writes one object to --out.

    python tools/bench_scenario_exposure.py [--ks 8,66] [--reps 2] [--out profiles/h100_scenario_exposure.json]
    python tools/bench_scenario_exposure.py --sweep-only --ks 66     # the plain sweep alone (any build of the library)

Cluster: synth.make_rebalance(4) (1 048 576 partitions x 1 024 nodes) with its own node changes cleared; scenario j
takes live node j out.  Schedules at MaxConcurrentPartitionMovesPerNode 1, 2 and 4, for both favor_min_nodes.

  arm 1  one sweep call with the schedules: without an exposure, with one without dom peaks, with one with them,
         alternating, `reps` times each;
  arm 2  the one-by-one path for `samples` scenarios, scaled to K: their next rows copied out (one sweep call with
         want_rows), then per (scenario, count) the begMap tables built on the host, blance_moves_create,
         blance_moves_schedule and blance_moves_exposure.  Its exposures are checked equal to the sweep's.

Timings are host wall clock around calls that end in a device synchronise; wave sizes, device bytes and the
exposure's device time come from the library's BLANCE_SCENARIO_TIMES report (CUDA events).  --sweep-only times the
plain sweep (arm 1 without the exposure) and calls nothing an older build of the package lacks, so a copy of this
script in another build's tools/ compares the two builds in alternating processes."""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

from bench_chains import clocks  # noqa: E402
from bench_scenarios import CaptureStderr, gpu_info, parse_waves  # noqa: E402

from blance_b200 import synth, tables  # noqa: E402

COUNTS = [1, 2, 4]
EXPO_RE = re.compile(r"exposure ([\d.]+) ms \((\d+) device bytes\)")


def scenarios(t, k):
    live = [q for q in range(t.n_nodes) if not t.node_removed[q]][:k]
    out = []
    for j in live:
        rm = np.zeros(t.n_node_ids, np.uint8)
        rm[j] = 1
        out.append(dict(node_removed=rm, node_added=np.zeros(t.n_node_ids, np.uint8), add_is_nil=0))
    return out


def sweep(ctx, t, scs, favor, exposure=None, want_rows=()):
    kw = {} if exposure is None else dict(exposure=exposure)
    with CaptureStderr() as cap:
        t0 = time.perf_counter()
        res = ctx.plan_scenarios(t, scs, favor, want_rows=want_rows, schedule=COUNTS, **kw)
        s = time.perf_counter() - t0
    info = parse_waves(cap.text)
    ex = EXPO_RE.findall(cap.text)
    info.update(exposure_ms=round(sum(float(m[0]) for m in ex), 3), exposure_bytes=sum(int(m[1]) for m in ex))
    return res, s, info


def one_by_one(ctx, t, scs, favor, samples):
    """(seconds per scenario, exposures [samples][counts]) of the one-by-one path."""
    import scenario_exposure_ref as REF
    t0 = time.perf_counter()
    res = ctx.plan_scenarios(t, scs[:samples], favor, want_rows=range(samples), schedule=COUNTS)
    mover = (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8)
    cons = np.asarray(t.state_constraints, np.int32)
    got = []
    for i in range(samples):
        st = tables.scenario_tables(t, scs[i])
        member, beg, end = REF.begmap_rows(st, res[i].next_rows)
        row = []
        for c in COUNTS:
            h, _ = ctx.moves_create(st.state_slot_off, beg, end, favor, st.n_node_ids)
            ctx.moves_schedule(h, c, mover)
            e = ctx.moves_exposure(h, cons, st.top_state)
            ctx.moves_free(h)
            for k, fill, dt in REF.PART_FILL:
                full = np.full(st.n_parts, fill, dt)
                full[member] = e[k]
                e[k] = full
            row.append(e)
        got.append(row)
    return (time.perf_counter() - t0) / samples, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="8,66")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--samples", type=int, default=2)
    ap.add_argument("--sweep-only", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = tables.Context()
    t = synth.make_rebalance(4)
    t.node_removed[:] = 0
    t.node_added[:] = 0
    rec = dict(workload="cfg 4 (1 048 576 partitions x 1 024 nodes), K single live-node failures, schedules at counts 1, 2, 4",
               **gpu_info(), **clocks(), runs=[])
    for k in [int(x) for x in args.ks.split(",")]:
        scs = scenarios(t, k)
        for favor in (False, True):
            sweep(ctx, t, scs[:1], favor)                               # warm-up
            if args.sweep_only:
                runs = [sweep(ctx, t, scs, favor) for _ in range(args.reps)]
                rec["runs"].append(dict(K=k, favor_min_nodes=favor, sweep_s=[round(r[1], 3) for r in runs], wave_size=runs[-1][2]["wave_size"],
                                        device_bytes_per_scenario=runs[-1][2]["device_bytes_per_scenario"]))
                print(json.dumps(rec["runs"][-1]), flush=True)
                continue
            arms = dict(none=None, no_dom=dict(series_cap=0, dom=False), dom=dict(series_cap=0, dom=True))
            sweep(ctx, t, scs[:1], favor, arms["dom"])
            times = {a: [] for a in arms}
            info = {}
            for _ in range(args.reps):
                for a, e in arms.items():
                    res, s, inf = sweep(ctx, t, scs, favor, e)
                    times[a].append(round(s, 3))
                    info[a] = inf
                    if a == "dom":
                        dom_res = res
            per, ones = one_by_one(ctx, t, scs, favor, min(args.samples, k))
            for i, row in enumerate(ones):
                for c, e in enumerate(row):
                    d = dom_res[i].exposures[c]
                    for f in ("rounds", "peak", "peak_round", "area", "dom_peak", "dom_peak_round", "part_min_copies", "part_no_top", "part_flags"):
                        assert np.array_equal(np.asarray(d[f]), np.asarray(e[f])), (k, favor, i, c, f)
            best = {a: min(v) for a, v in times.items()}
            worst = [dict(count=c, peak={m: int(max(r.exposures[x]["peak"][mi] for r in dom_res))
                                         for mi, m in enumerate(("NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY"))},
                          dom_peak_max=int(max(r.exposures[x]["dom_peak"].max() for r in dom_res)))
                     for x, c in enumerate(COUNTS)]
            rec["runs"].append(dict(
                K=k, favor_min_nodes=favor, sweep_s=times, wave_size={a: info[a]["wave_size"] for a in arms},
                device_bytes_per_scenario={a: info[a]["device_bytes_per_scenario"] for a in arms},
                exposure_ms={a: info[a]["exposure_ms"] for a in ("no_dom", "dom")},
                exposure_bytes_after_schedule={a: info[a]["exposure_bytes"] for a in ("no_dom", "dom")},
                exposure_share_of_sweep={a: round((best[a] - best["none"]) / best[a], 4) for a in ("no_dom", "dom")},
                one_by_one_s_per_scenario=round(per, 3), one_by_one_measured=min(args.samples, k),
                one_by_one_scaled_s=round(per * k, 3), speedup_vs_one_by_one=round(per * k / best["dom"], 2),
                sampled_exposures_equal=min(args.samples, k) * len(COUNTS), worst_over_scenarios=worst))
            print(json.dumps(rec["runs"][-1]), flush=True)
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
