"""BASELINE config 5 - 1 024 independent PlanNextMapEx instances (multi-tenant rebalance fan-out) - over 1/2/4/8 GPUs of
one node through ONE multi-device context (blance_ctx_create_multi): the library shards instance i -> device i mod G,
one host thread per device, no collective.  The struct arrays are built once; the timed call is
blance_plan_next_map_batch alone (host buffers: H2D, all kernels, D2H inside).  Every instance of the last run is
compared with the array oracle on 32 sampled instances (the -m gpu test checks all of a 160-instance batch).

    python tools/bench_cfg5.py [--gpus 1,2,4,8] [--instances 1024] > cfg5_scale.json
"""
import argparse, ctypes, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from blance_b200 import synth, tables
from oracle_loader import fast_lib_path

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", default="1")
ap.add_argument("--instances", type=int, default=1024)
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
FAST = ctypes.CDLL(fast_lib_path())
FAST.oracle_fast_plan_next_map.argtypes = [ctypes.c_void_p, ctypes.c_void_p]

def oracle(t):
    r = tables.PlanResult(t); s = t.struct()
    assert FAST.oracle_fast_plan_next_map(ctypes.byref(s), ctypes.byref(r.out)) == 0
    return r

n = args.instances
ctx1 = tables.Context(0)
fresh = [synth.make_fresh(5, seed_offset=i) for i in range(n)]
got = ctx1.run_batch(ctx1.prepare_batch(fresh))
rebs = [synth.make_rebalance(5, g.next_rows, seed_offset=i) for i, g in enumerate(got)]
ctx1.close()
parts = sum(t.n_parts for t in rebs)
rows = []
for G in [int(x) for x in args.gpus.split(",")]:
    ctx = tables.Context(device_ids=list(range(G)))
    prep = ctx.prepare_batch(rebs)
    ctx.run_batch(prep)
    ts = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        res = ctx.run_batch(prep)
        ts.append(time.perf_counter() - t0)
    ok = all(np.array_equal(res[i].next_rows, oracle(rebs[i]).next_rows) for i in range(0, n, max(1, n // 32)))
    rows.append({"n_gpus": G, "instances": n, "partitions": parts, "best_ms": 1e3 * min(ts), "median_ms": 1e3 * sorted(ts)[len(ts) // 2],
                 "partitions_per_s": parts / min(ts), "instances_per_s": n / min(ts), "sampled_instances_equal_oracle": bool(ok)})
    ctx.close()
base = rows[0]["partitions_per_s"] / rows[0]["n_gpus"]
for r in rows:
    r["scaling_efficiency_vs_first_row"] = r["partitions_per_s"] / (base * r["n_gpus"])
print(json.dumps({"workload": "cfg5: %d instances of 1024 partitions x 64 nodes (rack rules), rebalance stage" % n,
                  "api": "blance_ctx_create_multi + blance_plan_next_map_batch, host buffers, wall clock of the C call", "rows": rows}, indent=1))
