"""Times the map audit (include/blance_b200.h, "auditing a partition map") on an H100.

1. The headline map alone (cfg 4: 1 048 576 partitions x 1 024 nodes, nodes only), resident on the device
   (blance_plan_audit: no copy of the rows), with and without the failover matrix, alternating.  The time is a host
   clock around the call, which ends in a stream synchronise; it includes the call's allocation and its copy-out
   (4 MB for the matrix).  Next to it the time of the audit kernels alone (CUDA events around them,
   blance_audit_out.kernel_ms) and the rows they stream (partitions x padded slots x 4 bytes) over that time.
2. What-if sweeps with and without the audit, alternating, against the alternative without it: the rows of every
   scenario copied out and walked on the host with numpy (nodes-only counts: copies, top copies and the failover
   matrix; the hierarchy-rule check has no numpy form here and is left out of the host arm, which therefore
   UNDERSTATES the alternative).  A cfg 3 rack-failure sweep (rules, full-width masks) and cfg 4 node-failure sweeps
   (--k4 takes a list; the host arm is left out above --host-cap scenarios).  Each sweep also reports the audit
   kernels' own time per wave (events), which is what the audit adds to the wave's device time.

The card's name, power limit and SM clocks are read in the same run.  Prints one JSON object; --out also writes it.

    python tools/bench_audit.py [--reps 9] [--k3 8] [--k4 8,66] [--p3 65536] [--out audit.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from blance_b200 import synth, tables  # noqa: E402


def hardware():
    import torch
    hw = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        hw["power_limit"], hw["sm_clock"], hw["sm_clock_max"] = [x.strip() for x in q.split(",")]
    except (OSError, ValueError, subprocess.TimeoutExpired):
        hw["nvidia_smi"] = "unavailable"
    return hw


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def med(xs):
    return round(statistics.median(xs), 3)


def headline(ctx, reps):
    t = synth.make_rebalance(4)
    plan = ctx.upload(t)
    arms = {"plain": dict(n2n=False), "n2n": dict(n2n=True)}
    for kw in arms.values():                                   # warm-up of both shapes
        for _ in range(2):
            ctx.plan_audit(plan, t, **kw)
    ms = {k: [] for k in arms}
    kms = {k: [] for k in arms}
    for _ in range(reps):
        for k, kw in arms.items():
            dt, r = timed(lambda: ctx.plan_audit(plan, t, **kw))
            ms[k].append(dt)
            kms[k].append(r.kernel_ms)
    got = ctx.plan_audit(plan, t, n2n=True)
    assert np.array_equal(got.dom_copies, np.bincount(np.asarray(t.cur_rows).reshape(-1), minlength=t.n_nodes))
    ctx.free(plan)
    row_bytes = t.n_parts * max(4, (t.n_slots + 3) // 4 * 4) * 4
    out = {"partitions": t.n_parts, "nodes": t.n_nodes, "row_bytes_streamed": row_bytes, "reps": reps}
    for k in arms:
        out[k + "_ms_median"] = med(ms[k])
        out[k + "_ms_min_max"] = [round(min(ms[k]), 3), round(max(ms[k]), 3)]
        out[k + "_kernels_ms_median"] = med(kms[k])
        out[k + "_kernels_ms_min_max"] = [round(min(kms[k]), 4), round(max(kms[k]), 4)]
        out[k + "_row_GBps_kernels"] = round(row_bytes / (statistics.median(kms[k]) * 1e-3) / 1e9, 1)
    return out


def numpy_walk(t, rows):
    """The nodes-only counts of one final map on the host."""
    N = t.n_nodes
    rows = rows.reshape(t.n_parts, -1)
    copies = np.bincount(rows[rows >= 0], minlength=t.n_node_ids)
    top = np.bincount(rows[rows[:, 0] >= 0, 0], minlength=t.n_node_ids)
    n2n = np.zeros(N * N, np.int64)
    for c in range(1, rows.shape[1]):
        sel = (rows[:, c] >= 0) & (rows[:, 0] >= 0) & (rows[:, c] != rows[:, 0]) & (rows[:, c] < N) & (rows[:, 0] < N)
        n2n += np.bincount(rows[sel, 0].astype(np.int64) * N + rows[sel, c], minlength=N * N)
    return copies, top, n2n


def failures(t, groups):
    out = []
    for g in groups:
        rm = np.array(t.node_removed, np.uint8)
        rm[list(g)] = 1
        out.append(dict(node_removed=rm))
    return out


def sweep(ctx, name, t, scs, reps, host_arm=True):
    K = len(scs)
    arms = {"plain": lambda: ctx.plan_scenarios(t, scs, False),
            "audit": lambda: ctx.plan_scenarios(t, scs, False, audit=dict(n2n=True))}
    if host_arm:
        arms["rows_out_numpy"] = lambda: [numpy_walk(t, r.next_rows) for r in ctx.plan_scenarios(t, scs, False, want_rows=range(K))]
    ms = {k: [] for k in arms}
    res = {}
    for k, f in arms.items():
        f()                                                     # warm-up
    for _ in range(reps):
        for k, f in arms.items():
            dt, res[k] = timed(f)
            ms[k].append(dt)
    for r, (copies, top, n2n) in zip(res["audit"], res.get("rows_out_numpy", [])):      # all partitions are assigned here
        assert np.array_equal(r.audit.dom_copies, copies) and np.array_equal(r.audit.dom_top, top)
        assert np.array_equal(r.audit.n2n.reshape(-1), n2n)
    out = {"cluster": name, "partitions": t.n_parts, "nodes": t.n_nodes, "rules": int(t.n_rules) if t.has_hier_rules else 0,
           "scenarios": K, "reps": reps}
    for k in arms:
        out[k + "_ms_median"] = med(ms[k])
        out[k + "_ms_min_max"] = [round(min(ms[k]), 3), round(max(ms[k]), 3)]
    out["audit_over_plain_percent"] = round(100.0 * (statistics.median(ms["audit"]) / statistics.median(ms["plain"]) - 1.0), 2)
    # the audit kernels of the last timed sweep: one value per wave (its scenarios all carry it)
    waves = sorted({round(float(r.audit.kernel_ms), 4) for r in res["audit"]})
    out["audit_kernels_ms_per_wave"] = waves
    out["audit_kernels_percent_of_plain_sweep"] = round(100.0 * sum(waves) / statistics.median(ms["plain"]), 4)
    out["rule_miss_parts"] = [int(r.audit.rule_miss_parts) for r in res["audit"]]
    out["warn_parts"] = [int(r.warn_parts) for r in res["audit"]]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--k3", type=int, default=8, help="rack failures of the cfg 3 sweep")
    ap.add_argument("--k4", default="8", help="node failures of the cfg 4 sweeps, comma separated")
    ap.add_argument("--host-cap", type=int, default=8, help="largest sweep that also runs the rows-out + numpy arm")
    ap.add_argument("--p3", type=int, default=65536, help="partitions of the cfg 3 cluster")
    ap.add_argument("--sweep-reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    ctx = tables.Context()                                      # fails without a device: there is no other arm
    result = {"hardware": hardware(), "headline_audit": headline(ctx, a.reps), "sweeps": []}
    fresh = synth.make_fresh(3, P=a.p3)
    t3 = synth.make_rebalance(3, prev_rows=ctx.plan_next_map(fresh).next_rows, P=a.p3)
    result["sweeps"].append(sweep(ctx, "cfg3 rack failures", t3, failures(t3, [range(8 * r, 8 * r + 8) for r in range(1, a.k3 + 1)]), a.sweep_reps))
    t4 = synth.make_rebalance(4)
    for k4 in [int(x) for x in a.k4.split(",")]:
        result["sweeps"].append(sweep(ctx, "cfg4 node failures", t4, failures(t4, [[16 + j] for j in range(k4)]), a.sweep_reps, k4 <= a.host_cap))
    ctx.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
