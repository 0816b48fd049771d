"""What-if sweeps through blance_plan_scenarios against the same scenarios planned one by one with
blance_plan_next_map, alternating in the same process, with sampled correctness checks.  Prints one JSON object
and writes it to --out.

    python tools/bench_scenarios.py [--ks 1,8,33,66,132] [--cfgs 4,3] [--out profiles/h100_scenarios.json]
    python tools/bench_scenarios.py --sweep stickiness,replicas [--out profiles/h100_option_sweeps.json]
    python tools/bench_scenarios.py --schedule 1,2,4 [--ks 8,66] [--cap 4] [--out profiles/h100_scenario_schedule.json]

--schedule times, on cfg 4 node-failure sweeps, the plain sweep (blance_plan_scenarios), the sweep with the
rebalance schedules at those MaxConcurrentPartitionMovesPerNode values (blance_plan_scenarios_schedule) and the
only alternative without it (rows copied out, then blance_moves_create + blance_moves_schedule per scenario and per
value), alternating in one process.  The alternative runs on the first --cap scenarios and is extrapolated to K.
Sampled scenarios' schedule summaries are checked against the serial oracle (tests/schedule_oracle.c).  It also
times the wave engine as a wave of one on the headline rebalance next to blance_moves_schedule on the same moves.

--sweep plans option variants of the cfg 4 cluster instead (StateStickiness {0, 1, 2, 3, 5, 8}, or replicas
{1, 2, 3, 4} on a base widened to 4 replica slots) through blance_plan_scenarios_ex, against the same variants one
by one, and checks every variant's plan against its one-by-one plan.

Clusters: synth.make_rebalance(4) (1 M partitions x 1 024 nodes) and synth.make_rebalance(3) (65 536 x 256 with
zone and rack rules; its previous map is the fresh stage's plan).  Scenario j keeps the configuration's own
removals and additions and also fails live node j; cfg 3 adds one scenario per rack that fails the whole rack.
Timings are host wall clock around calls that end in a device synchronise; the wave size, device bytes per
scenario and the summary kernel's time come from the library's BLANCE_SCENARIO_TIMES report (CUDA events)."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from blance_b200 import synth, tables  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.splitlines()[0].split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as e:   # noqa: BLE001 - recorded, not fatal
        return dict(gpu="unknown (%s)" % e, power_limit="unknown")


class CaptureStderr:
    """Collects what the library writes to fd 2 (its BLANCE_SCENARIO_TIMES lines)."""

    def __enter__(self):
        sys.stderr.flush()
        self.f = tempfile.TemporaryFile(mode="w+")
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        os.environ["BLANCE_SCENARIO_TIMES"] = "1"
        return self

    def __exit__(self, *a):
        os.environ.pop("BLANCE_SCENARIO_TIMES", None)
        sys.stderr.flush()
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read()
        self.f.close()


WAVE_RE = re.compile(r"scenario wave at \d+: (\d+) scenarios \(wave size (\d+), (\d+) device bytes each\), ([\d.]+) ms, summary ([\d.]+) ms")


def parse_waves(text):
    waves = [dict(n=int(m[0]), wave=int(m[1]), bytes=int(m[2]), ms=float(m[3]), summary_ms=float(m[4])) for m in WAVE_RE.findall(text)]
    return dict(wave_size=max(w["wave"] for w in waves) if waves else None, waves=len(waves),
                device_bytes_per_scenario=waves[0]["bytes"] if waves else None,
                wave_ms=round(sum(w["ms"] for w in waves), 3), summary_ms=round(sum(w["summary_ms"] for w in waves), 3))


def live_nodes(t):
    return [q for q in range(t.n_nodes) if not t.node_removed[q] and not t.node_added[q]]


def failure_scenarios(t, k):
    out = []
    for q in live_nodes(t)[:k]:
        rm = t.node_removed.copy()
        rm[q] = 1
        out.append(dict(node_removed=rm))
    return out


def rack_scenarios(t, rack=8):
    out = []
    for r in range(t.n_nodes // rack):
        rm = t.node_removed.copy()
        rm[r * rack:(r + 1) * rack] = 1
        out.append(dict(node_removed=rm))
    return out


def sweep(ctx, t, scs, max_concurrent=0):
    with CaptureStderr() as cap:
        t0 = time.perf_counter()
        res = ctx.plan_scenarios(t, scs, False, max_concurrent=max_concurrent)
        wall = time.perf_counter() - t0
    return res, wall, parse_waves(cap.text)


def one_by_one(ctx, t, scs):
    t0 = time.perf_counter()
    outs = [ctx.plan_next_map(tables.scenario_tables(t, sc)) for sc in scs]
    return outs, time.perf_counter() - t0


def numpy_summary(ctx, t, next_rows):
    """The summaries recomputed on the host from the flat tables (moves from blance_calc_partition_moves)."""
    a = t.part_in_assign != 0
    beg = np.where((t.part_in_prev != 0)[:, None], t.prev_rows, -1)[a]
    node, _state, kind, count = ctx.calc_partition_moves(t.state_slot_off, beg, next_rows[a], False)
    valid = np.arange(node.shape[1])[None, :] < count[:, None]
    ops = np.zeros((t.n_node_ids, 4), np.int64)
    np.add.at(ops, (node[valid], kind[valid]), 1)
    final = np.where(a[:, None], next_rows, t.prev_rows)
    w = np.where((t.has_part_weights != 0) & (t.part_has_weight != 0), t.part_weight, 1).astype(np.int64)
    load = np.zeros((t.n_states, t.n_node_ids), np.int64)
    for s in range(t.n_states):
        blk = final[:, t.state_slot_off[s]:t.state_slot_off[s + 1]]
        ok = blk >= 0
        load[s] = np.bincount(blk[ok], weights=np.broadcast_to(w[:, None], blk.shape)[ok], minlength=t.n_node_ids).astype(np.int64)
    return ops, load, int((count > 0).sum()), int(count.sum())


def check_sample(ctx, t, scs, res, rng):
    """2 sampled scenarios: rows equal blance_plan_next_map on the substituted tables; summary equals numpy."""
    ok = True
    for i in sorted(set(rng.choice(len(scs), size=min(2, len(scs)), replace=False).tolist())):
        st = tables.scenario_tables(t, scs[i])
        ref = ctx.plan_next_map(st)
        got = ctx.plan_scenarios(t, [scs[i]], False, want_rows=[0])[0]
        ok &= bool(np.array_equal(got.next_rows, ref.next_rows) and np.array_equal(got.warn, ref.warn) and
                   (got.iters_run, got.converged, got.steps) == (ref.iters_run, ref.converged, ref.steps))
        ops, load, moved, total = numpy_summary(ctx, st, ref.next_rows)
        ok &= bool(np.array_equal(res[i].node_ops, ops) and np.array_equal(res[i].state_node_load, load) and
                   (res[i].parts_moved, res[i].ops_total) == (moved, total) and res[i].steps == ref.steps)
    return ok


def run_cfg(ctx, cfg, ks, rng):
    if cfg == 3:
        t = synth.make_rebalance(3, prev_rows=ctx.plan_next_map(synth.make_fresh(3)).next_rows)
    else:
        t = synth.make_rebalance(cfg)
    ctx.plan_scenarios(t, failure_scenarios(t, 2), False)            # warm-up of every kernel the sweep uses
    ctx.plan_next_map(t)
    rows = []
    for k in ks:
        scs = failure_scenarios(t, k) + (rack_scenarios(t) if cfg == 3 else [])
        res, wall_a, info = sweep(ctx, t, scs)
        _, serial = one_by_one(ctx, t, scs)
        _, wall_b, _ = sweep(ctx, t, scs)
        wall = min(wall_a, wall_b)
        row = dict(cfg=cfg, K=k, scenarios=len(scs), sweep_s=[round(wall_a, 3), round(wall_b, 3)],
                   scenarios_per_s=round(len(scs) / wall, 3), one_by_one_s=round(serial, 3),
                   one_by_one_scenarios_per_s=round(len(scs) / serial, 3), speedup=round(serial / wall, 3),
                   summary_share=round(info["summary_ms"] / info["wave_ms"], 5) if info["wave_ms"] else None,
                   correct=check_sample(ctx, t, scs, res, rng), **info)
        print(json.dumps(row), flush=True)
        rows.append(row)
    return t, rows


WAVE_SCHED_RE = re.compile(r"schedule ([\d.]+) ms")


def schedule_summary_of(off, node, kind, n_node_ids, c, mover):
    """The serial oracle's schedule at count c, reduced to the summaries of blance_plan_scenarios_schedule."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import schedule_oracle as SO
    from test_scenario_schedule import schedule_summaries
    ro, so, _ = SO.schedule(off, node, kind, n_node_ids, c, mover)
    return schedule_summaries(off, node, n_node_ids, ro, so)


def scenario_moves(ctx, t, next_rows):
    """The CSR move lists the scenario schedule runs over (blance_moves_create on beg / end rows)."""
    a = t.part_in_assign != 0
    beg = np.where(((t.part_in_prev != 0) & a)[:, None], t.prev_rows, -1).astype(np.int32)
    beg[~a] = next_rows[~a]
    return beg


def run_schedule_sweeps(ctx, counts, ks, cap, rng):
    t = synth.make_rebalance(4)
    mover = (np.arange(t.n_node_ids) < t.n_nodes).astype(np.uint8)
    warm = failure_scenarios(t, 2)
    ctx.plan_scenarios(t, warm, False)                                     # warm-up of every kernel the runs use
    ctx.plan_scenarios(t, warm, False, schedule=counts)
    rows = []
    for k in ks:
        scs = failure_scenarios(t, k)

        def timed(**kw):
            with CaptureStderr() as cap_err:
                t0 = time.perf_counter()
                res = ctx.plan_scenarios(t, scs, False, **kw)
                wall = time.perf_counter() - t0
            return res, wall, parse_waves(cap_err.text), sum(float(x) for x in WAVE_SCHED_RE.findall(cap_err.text))

        def alternative():
            n = min(cap, len(scs))
            t0 = time.perf_counter()
            res = ctx.plan_scenarios(t, scs[:n], False, want_rows=range(n))
            t1 = time.perf_counter()
            out = []
            for r in res:
                h, _ = ctx.moves_create(t.state_slot_off, scenario_moves(ctx, t, r.next_rows), r.next_rows, False, t.n_node_ids)
                out.append([ctx.moves_schedule(h, c, mover)[2] for c in counts])
                ctx.moves_free(h)
            t2 = time.perf_counter()
            return n, t1 - t0, t2 - t1, out

        plain_a, plain_s_a, _, _ = timed()
        sched_a, sched_s_a, info, sched_ms_a = timed(schedule=counts)
        n_alt, alt_plan_s, alt_sched_s, _ = alternative()
        _, plain_s_b, _, _ = timed()
        _, sched_s_b, _, sched_ms_b = timed(schedule=counts)
        plain_s, sched_s = min(plain_s_a, plain_s_b), min(sched_s_a, sched_s_b)
        # the alternative at K: the plain sweep with rows out, plus the per-scenario schedules extrapolated from n_alt
        alt_s = plain_s + alt_sched_s * len(scs) / n_alt
        ok = True
        for i in sorted(set(rng.choice(len(scs), size=min(2, len(scs)), replace=False).tolist())):
            r = ctx.plan_scenarios(t, [scs[i]], False, want_rows=[0])[0]
            h, total = ctx.moves_create(t.state_slot_off, scenario_moves(ctx, t, r.next_rows), r.next_rows, False, t.n_node_ids)
            off, node, _, kind = ctx.moves_fetch(h, total)
            ctx.moves_free(h)
            for c, s in zip(counts, sched_a[i].schedules):
                want = schedule_summary_of(off, node, kind, t.n_node_ids, c, mover)
                ok &= all(getattr(s, f) == want[f] for f in ("rounds", "moves_done", "stuck_parts", "max_batch"))
                ok &= all(np.array_equal(getattr(s, f), want[f]) for f in ("node_rounds", "node_last_round", "part_done_round"))
            ok &= bool(sched_a[i].ops_total == plain_a[i].ops_total == r.ops_total)
        row = dict(cfg=4, K=k, counts=counts, plain_sweep_s=[round(plain_s_a, 3), round(plain_s_b, 3)],
                   schedule_sweep_s=[round(sched_s_a, 3), round(sched_s_b, 3)],
                   schedule_device_ms=[round(sched_ms_a, 3), round(sched_ms_b, 3)],
                   added_over_plain=round((sched_s - plain_s) / plain_s, 4),
                   alternative=dict(scenarios_measured=n_alt, plan_with_rows_s=round(alt_plan_s, 3),
                                    schedules_s=round(alt_sched_s, 3), extrapolated_to_K_s=round(alt_s, 3)),
                   speedup_vs_alternative=round(alt_s / sched_s, 3), rounds=[[s.rounds for s in r.schedules] for r in sched_a[:4]],
                   correct=bool(ok), **info)
        print(json.dumps(row), flush=True)
        rows.append(row)
    # the wave engine as a wave of one on the headline rebalance, next to blance_moves_schedule on the same moves
    one = []
    r = ctx.plan_scenarios(t, [{}], False, want_rows=[0])[0]
    h, _ = ctx.moves_create(t.state_slot_off, scenario_moves(ctx, t, r.next_rows), r.next_rows, False, t.n_node_ids)
    for c in counts:
        ms = []
        for _ in range(2):
            with CaptureStderr() as cap_err:
                w = ctx.plan_scenarios(t, [{}], False, schedule=[c])[0].schedules[0]
            ms.append(float(WAVE_SCHED_RE.findall(cap_err.text)[0]))
        dev = [ctx.moves_schedule(h, c, mover)[2] for _ in range(2)]
        one.append(dict(c=c, rounds=w.rounds, wave_of_one_ms=[round(x, 3) for x in ms],
                        moves_schedule_ms=[round(d["device_ms"], 3) for d in dev], same_rounds=dev[0]["rounds"] == w.rounds,
                        same_max_batch=dev[0]["max_batch"] == w.max_batch))
        print(json.dumps(one[-1]), flush=True)
    ctx.moves_free(h)
    return dict(sweeps=rows, headline_wave_of_one=one)


def option_variants(t, kind):
    """The option sweeps of the 1 M x 1 024 cluster (blance_scenario_opts as dicts): StateStickiness of every state
    in {0, 1, 2, 3, 5, 8}, or the replica count in {1, 2, 3, 4} on a base widened to 4 replica slots."""
    S = t.n_states
    if kind == "stickiness":
        vals = [0, 1, 2, 3, 5, 8]
        return t, [dict(state_stickiness=np.full(S, v, np.int32), state_has_stickiness=np.ones(S, np.uint8)) for v in vals], vals
    vals = [1, 2, 3, 4]
    w = tables.widen_layout(t, [int(t.state_constraints[0]), max(vals)])
    return w, [dict(state_constraints=np.array([t.state_constraints[0], v], np.int32)) for v in vals], vals


def run_option_sweep(ctx, kind):
    """K option variants as one blance_plan_scenarios_ex call against the same variants planned one by one with
    blance_plan_next_map, alternating (sweep, one by one, sweep).  Every variant's rows, warnings, iterations and
    steps are compared with its one-by-one plan."""
    t, opts, vals = option_variants(synth.make_rebalance(4), kind)
    scs = [{} for _ in opts]
    ctx.plan_scenarios(t, scs[:2], False, opts=opts[:2])               # warm-up of every kernel the sweep uses
    ctx.plan_next_map(tables.scenario_tables(t, {}, opts[0]))

    def sweep_once():
        with CaptureStderr() as cap:
            t0 = time.perf_counter()
            res = ctx.plan_scenarios(t, scs, False, want_rows=range(len(scs)), opts=opts)
            wall = time.perf_counter() - t0
        return res, wall, parse_waves(cap.text)
    res, wall_a, info = sweep_once()
    t0 = time.perf_counter()
    serial = [ctx.plan_next_map(tables.scenario_tables(t, {}, o)) for o in opts]
    serial_s = time.perf_counter() - t0
    _, wall_b, _ = sweep_once()
    wall = min(wall_a, wall_b)
    same = [bool(np.array_equal(r.next_rows, s.next_rows) and np.array_equal(r.warn, s.warn) and
                 (r.iters_run, r.converged, r.steps) == (s.iters_run, s.converged, s.steps)) for r, s in zip(res, serial)]
    variants = [dict(value=v, matches_one_by_one=ok, iterations=r.iters_run, steps=r.steps, sticky_steps=r.sticky_steps,
                     sticky_share=round(r.sticky_steps / r.steps, 4) if r.steps else None, parts_moved=r.parts_moved,
                     ops_total=r.ops_total, warn_parts=r.warn_parts, one_by_one_device_ms=round(s.device_ms, 3),
                     one_by_one_pass_ms=round(s.pass_ms, 3)) for v, r, s, ok in zip(vals, res, serial, same)]
    row = dict(sweep=kind, cfg=4, K=len(opts), n_slots=t.n_slots, sweep_s=[round(wall_a, 3), round(wall_b, 3)],
               one_by_one_s=round(serial_s, 3), speedup=round(serial_s / wall, 3), correct=all(same),
               variants=variants, **info)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,8,33,66,132")
    ap.add_argument("--cfgs", default="4,3")
    ap.add_argument("--wave-ks", default="33,66,132", help="explicit max_concurrent values tried on cfg 4 at the largest K")
    ap.add_argument("--sweep", default=None, help="option sweeps instead of node failures: stickiness, replicas, or both (comma separated)")
    ap.add_argument("--schedule", default=None, help="MaxConcurrentPartitionMovesPerNode values, e.g. 1,2,4: time the sweeps with schedules")
    ap.add_argument("--cap", type=int, default=4, help="--schedule: scenarios the one-by-one alternative runs on before extrapolating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    rng = np.random.default_rng(0)
    rec = dict(tool="tools/bench_scenarios.py", **gpu_info())
    ctx = tables.Context()
    if a.schedule:
        rec["schedule"] = run_schedule_sweeps(ctx, [int(x) for x in a.schedule.split(",")],
                                              [int(x) for x in (a.ks if a.ks != ap.get_default("ks") else "8,66").split(",")], a.cap, rng)
        rec["command"] = "python tools/bench_scenarios.py " + " ".join(sys.argv[1:])
        ctx.close()
        print(json.dumps(rec))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(rec, f, indent=1)
        return
    if a.sweep:
        rec["option_sweeps"] = [run_option_sweep(ctx, kind) for kind in a.sweep.split(",")]
        ctx.close()
        print(json.dumps(rec))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(rec, f, indent=1)
        return
    rec["sm_count_note"] = "auto wave: free device memory, and at most sm_count / 2 above 768 nodes"
    rec["results"] = []
    for cfg in [int(x) for x in a.cfgs.split(",")]:
        t, rows = run_cfg(ctx, cfg, ks, rng)
        rec["results"] += rows
        if cfg == 4 and a.wave_ks:
            scs = failure_scenarios(t, max(ks))
            waves = []
            for mc in [0] + [int(x) for x in a.wave_ks.split(",")]:
                _, wall, info = sweep(ctx, t, scs, max_concurrent=mc)
                waves.append(dict(max_concurrent=mc, sweep_s=round(wall, 3), scenarios_per_s=round(len(scs) / wall, 3), **info))
                print(json.dumps(waves[-1]), flush=True)
            rec["cfg4_wave_sizes"] = dict(K=max(ks), runs=waves)
    ctx.close()
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
