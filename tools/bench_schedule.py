"""Times blance_moves_schedule (the orchestrator's whole lock-step schedule on the device, include/blance_b200.h) on
the headline cluster (cfg 4: 1 048 576 partitions x 1 024 nodes, -16/+16 nodes, planned on the GPU) at
MaxConcurrentPartitionMovesPerNode c = 1, 2 and 4, against the only way to get the same schedule without it: a host
loop of one blance_moves_available call per round (P-wide scan + sort on the device, two host syncs, the node lists
copied out) with the picks of filterNextPlausibleMovesForNode replayed on the host.

The host loop is capped at --host-rounds rounds per repetition and extrapolated linearly to the schedule's R (its
rounds get cheaper as partitions finish, so the extrapolation overstates it somewhat); the capped rounds are
checked op for op against the device schedule.  Device and host loop alternate, after a warm-up of each.  Every
device schedule is checked against the serial oracle (tests/schedule_oracle.c).  The card's name, power limit and
SM clocks are read in the same run.  Prints one JSON object; --out also writes it to a file.

    python tools/bench_schedule.py [--reps 5] [--host-rounds 40] [--out schedule.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import schedule_oracle as SO  # noqa: E402
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


def host_loop(ctx, h, off, kind, c, max_rounds):
    """One blance_moves_available call per round, picks replayed on the host; returns (sched_op of the rounds run,
    rounds run, seconds)."""
    P = len(off) - 1
    nxt = np.zeros(P, np.int32)
    count = max(1, c)
    out = []
    t0 = time.perf_counter()
    for _ in range(max_rounds):
        node_off, node_parts, best = ctx.moves_available(h, nxt)
        if node_off[-1] == 0:
            break
        picked = []
        for n in np.nonzero(np.diff(node_off))[0]:
            arr = node_parts[node_off[n]:node_off[n + 1]].tolist()
            if count == 1:
                picks = [int(best[n])]
            else:
                w = [SO.WEIGHT[int(kind[off[p] + nxt[p]])] for p in arr]
                picks = []
                for _ in range(min(count, len(arr))):
                    r = w.index(min(w))                 # the first index of the lowest weight
                    picks.append(arr[r])
                    arr[r], w[r] = arr[-1], w[-1]
                    arr.pop(); w.pop()
            picked += picks
        picked = np.asarray(picked, np.int64)
        out.append(off[picked] + nxt[picked])
        nxt[picked] += 1
    secs = time.perf_counter() - t0
    return (np.concatenate(out) if out else np.zeros(0, np.int64)), len(out), secs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=40)
    ap.add_argument("--parts", type=int, default=None, help="smaller cluster (rehearsal); default the headline size")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    hw = hardware()
    ctx = tables.Context()
    t = synth.make_rebalance(4, P=args.parts)
    plan = ctx.plan_next_map(t)
    h, total = ctx.moves_create(t.state_slot_off, t.prev_rows, plan.next_rows, False, t.n_node_ids)
    off, node, _, kind = ctx.moves_fetch(h, total)
    res = {"workload": "cfg4 rebalance moves (prev rows -> GPU-planned next rows)", "n_parts": t.n_parts,
           "n_nodes": t.n_nodes, "total_ops": total, "hardware": hw, "reps": args.reps,
           "host_rounds_cap": args.host_rounds, "per_c": {}}
    for c in (1, 2, 4):
        ro, so, sc = ctx.moves_schedule(h, c)                        # warm-up (and the result that is checked)
        t0 = time.perf_counter()
        want_ro, want_so, want = SO.schedule(off, node, kind, t.n_node_ids, c)
        oracle_s = time.perf_counter() - t0
        equal = bool(np.array_equal(ro, want_ro) and np.array_equal(so, want_so) and all(sc[k] == want[k] for k in want))
        host_loop(ctx, h, off, kind, c, 2)                          # warm-up of the host loop
        dev_ms, dev_wall_ms, host_ms_per_round, host_equal = [], [], [], True
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r2 = ctx.moves_schedule(h, c)
            dev_wall_ms.append((time.perf_counter() - t0) * 1e3)
            dev_ms.append(r2[2]["device_ms"])
            host_equal &= bool(np.array_equal(r2[0], ro) and np.array_equal(r2[1], so))
            hs, n_r, secs = host_loop(ctx, h, off, kind, c, args.host_rounds)
            host_ms_per_round.append(secs * 1e3 / max(n_r, 1))
            host_equal &= bool(np.array_equal(hs, so[:ro[n_r]]))
        R = sc["rounds"]
        res["per_c"][str(c)] = {
            "rounds": R, "moves_done": sc["moves_done"], "stuck_parts": sc["stuck_parts"], "max_batch": sc["max_batch"],
            "equal_oracle": equal, "oracle_seconds": round(oracle_s, 2),
            "device_ms_median": float(np.median(dev_ms)), "device_ms_all": [round(x, 3) for x in dev_ms],
            "device_call_wall_ms_median": float(np.median(dev_wall_ms)),
            "host_loop_ms_per_round_median": float(np.median(host_ms_per_round)),
            "host_loop_ms_extrapolated": float(np.median(host_ms_per_round)) * R,
            "host_loop_rounds_equal_device": host_equal,
        }
        print(json.dumps({str(c): res["per_c"][str(c)]}), flush=True)
    ctx.moves_free(h)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
