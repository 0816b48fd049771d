"""The values that feed the score at their extremes, on the CPU.

1. The count bound (include/blance_b200.h, blance_plan_in_check): the device keeps every node's weighted count in
   int32, the reference in 64-bit ints, so an instance with
       sum_p |w_p| * max(1, n_slots) + max_n max(|extra_tot_first[n]|, |extra_tot_rest[n]|) > INT32_MAX
   is refused as unsupported by blance_plan_in_check, by the host interning and by the scenario entry points
   (each scenario with its own weights and non-model counts).  Exactly at the bound is accepted, one more is not,
   with and without non-model counts.
2. The literal oracle equals the array-form oracle on randgen's instances with extreme values: partition weights
   of -10^9 .. 999 999 999, node weights of -2^31 .. 2^31 - 1 with and without the booster, StateStickiness of
   -5, 0 and 2^31 - 1.  This is what entitles the array-form oracle to judge the GPU at these values
   (test_value_range_gpu.py).
CPU only."""
import copy
import ctypes
import random

import numpy as np
import pytest

from oracle_loader import literal
from randgen import random_instance
from test_fast_oracle import FAST

from blance_b200 import BlanceError, _host, abi, tables

OK, INVALID, UNSUPPORTED = 0, -1, -2
I32_MAX = 2**31 - 1
BOUND_MSG = "exceeds int32"

L = literal()


# ---- 1. the count bound ---------------------------------------------------------------------------------------

def weighted(weights, ks=(1,), n_nodes=4):
    """PlanTables of len(weights) partitions, every one weighted, states with constraints ks (n_slots = sum(ks))."""
    t = tables.PlanTables(n_nodes, len(ks), len(weights), list(range(len(ks))), list(ks))
    t.has_part_weights = 1
    t.part_has_weight[:] = 1
    t.part_weight[:] = weights
    return t


BOUND_CASES = [  # (n_slots, non-model count); 2^31 - 1 is prime, so with 7 slots the count takes the remainder
    (1, 0), (1, 5), (1, -5), (7, 1), (7, -8)]


def bound_tables(n_slots, extra, over, which="first"):
    """PlanTables with sum |w| * n_slots + |extra| == INT32_MAX + over: weights alternate +-999 999 999 and the
    count of a non-model state (extra_tot_<which>, the sign of `extra`) sits on node 2."""
    left = (I32_MAX - abs(extra)) // n_slots
    ex = I32_MAX - left * n_slots
    w = []
    while left > 999999999:
        w.append(999999999 if len(w) % 2 == 0 else -999999999)
        left -= 999999999
    w.append(left)
    if ex == 0:
        w[-1] += over
    else:
        ex += over
    t = weighted(w, ks=(n_slots,))
    getattr(t, "extra_tot_" + which)[2] = ex if extra >= 0 else -ex
    return t


def check(t):
    msg = ctypes.create_string_buffer(256)
    s = t.struct()
    return abi.capi().blance_plan_in_check(ctypes.byref(s), msg, 256), msg.value.decode()


@pytest.mark.parametrize("n_slots,extra", BOUND_CASES)
@pytest.mark.parametrize("which", ["first", "rest"])
def test_plan_in_check_count_bound(n_slots, extra, which):
    assert check(bound_tables(n_slots, extra, 0, which)) == (OK, "")
    st, why = check(bound_tables(n_slots, extra, 1, which))
    assert st == UNSUPPORTED and BOUND_MSG in why


def test_plan_in_check_bound_counts_one_per_partition_without_weights():
    """Without has_part_weights every partition counts 1 whatever part_weight holds."""
    t = weighted([999999999] * 4, ks=(1,))
    t.has_part_weights = 0
    t.extra_tot_first[0] = I32_MAX - 4
    assert check(t) == (OK, "")
    t.extra_tot_rest[1] = -(I32_MAX - 3)
    assert check(t)[0] == UNSUPPORTED


def scenario_call(base, opts=None):
    """blance_plan_scenarios(_ex) of one scenario with a NULL context: the status and message of the argument
    checks (every scenario is checked before the context is used)."""
    lib = abi.capi()
    keep = []
    b = base.struct()
    scs = (abi.Scenario * 1)()
    for f in tables.SCENARIO_FIELDS:
        v = getattr(base, f)
        if f in ("add_is_nil", "has_node_weights"):
            setattr(scs[0], f, int(v))
            continue
        a = np.ascontiguousarray(v, dtype=np.int32 if f == "node_weight" else np.uint8)
        keep.append(a)
        setattr(scs[0], f, a.ctypes.data if a.size else None)
    outs = (abi.ScenarioOut * 1)()
    if opts is None:
        st = lib.blance_plan_scenarios(None, ctypes.byref(b), 1, scs, 0, 0, outs)
    else:
        ops = (abi.ScenarioOpts * 1)(tables._opts_struct(base, opts, keep))
        st = lib.blance_plan_scenarios_ex(None, ctypes.byref(b), 1, scs, ops, 0, 0, outs)
    return st, lib.blance_last_error(None).decode()


def scenario_ok(r):
    return r[0] == INVALID and "ctx is NULL" in r[1]


def scenario_refused(r):
    return r[0] == UNSUPPORTED and "scenario 0" in r[1] and BOUND_MSG in r[1]


@pytest.mark.parametrize("n_slots,extra", BOUND_CASES)
def test_scenario_count_bound_without_options(n_slots, extra):
    """No option touches the weights: the base's own bound decides, on both entry points."""
    for opts in (None, dict(state_stickiness=np.array([3], np.int32), state_has_stickiness=np.array([1], np.uint8))):
        assert scenario_ok(scenario_call(bound_tables(n_slots, extra, 0), opts))
        assert scenario_refused(scenario_call(bound_tables(n_slots, extra, 1), opts))


@pytest.mark.parametrize("n_slots,extra", BOUND_CASES)
def test_scenario_count_bound_with_weight_overrides(n_slots, extra):
    """The base is n_slots below the bound (its last partition one lighter); an override of that partition takes it to
    the bound or one weight unit beyond, and so do the non-model counts of an override."""
    base = bound_tables(n_slots, extra, 0)
    last = base.n_parts - 1
    w0 = int(base.part_weight[last])
    assert 0 < w0 < 999999999
    base.part_weight[last] = w0 - 1
    slack = n_slots
    assert scenario_ok(scenario_call(base))
    one = np.ones(1, np.uint8)
    part = np.array([last], np.int32)
    for w in (w0, -w0):
        assert scenario_ok(scenario_call(base, dict(has_part_weights=1, weight_overrides=(part, np.array([w], np.int32), one))))
    for w in (w0 + 1, -w0 - 1):
        assert scenario_refused(scenario_call(base, dict(has_part_weights=1, weight_overrides=(part, np.array([w], np.int32), one))))
    # the same base with one more unit of non-model count than its slack is refused through the override's extras
    ex = np.array(base.extra_tot_first)
    ex[3] = abs(int(ex[2])) + slack
    assert scenario_ok(scenario_call(base, dict(extra_tot_first=ex)))
    ex[3] += 1
    assert scenario_refused(scenario_call(base, dict(extra_tot_first=ex)))
    ex = np.array(base.extra_tot_rest)
    ex[1] = -(abs(int(base.extra_tot_first[2])) + slack + 1)
    assert scenario_refused(scenario_call(base, dict(extra_tot_rest=ex)))


def test_scenario_overrides_bring_a_base_within_the_bound():
    base = bound_tables(1, 0, 1)
    assert scenario_refused(scenario_call(base))
    part, one = np.zeros(1, np.int32), np.ones(1, np.uint8)
    assert scenario_ok(scenario_call(base, dict(has_part_weights=1, weight_overrides=(part, np.array([0], np.int32), one))))
    assert scenario_ok(scenario_call(base, dict(has_part_weights=0)))
    assert scenario_refused(scenario_call(base, dict(has_part_weights=1, weight_overrides=(part, np.array([-999999999], np.int32), one))))


def host_kwargs(w3, extra_weight):
    """String form: partitions 0, 1 of weight 999 999 999, partition 2 of weight `extra_weight` holding node a under
    the model state AND under the non-model state 'dead', partition 3 of weight w3, one slot: sum |w| + max extra =
    1 999 999 998 + 2 * |extra_weight| + |w3|."""
    prev = {"0": {"primary": ["a"]}, "1": {"primary": ["b"]}, "2": {"primary": ["a"], "dead": ["a"]}, "3": {}}
    return dict(prev_map=prev, partitions_to_assign={"3": {}}, nodes_all=["a", "b"], nodes_to_remove=[], nodes_to_add=[],
                model={"primary": (0, 1)}, partition_weights={"0": 999999999, "1": 999999999, "2": extra_weight, "3": w3})


@pytest.mark.parametrize("w3,extra_weight", [(147483649, 0), (-147483649, 0), (1, 73741824), (-1, -73741824)])
def test_host_interning_count_bound(w3, extra_weight):
    kw = host_kwargs(w3, extra_weight)
    ip = _host.intern_plan(**copy.deepcopy(kw))
    assert ip.in_ptr
    kw["partition_weights"]["3"] += 1 if w3 > 0 else -1
    with pytest.raises(BlanceError, match=BOUND_MSG):
        _host.intern_plan(**kw)


def wrapping_instance():
    """Node a holds the replica of h (weight 999 999 999) and two entries of h under states outside the model: its
    total is 2 999 999 997, which wraps in int32, while sum |w| x slots alone is 2 000 000 000."""
    prev = {"h": {"replica": ["a"], "x": ["a"], "y": ["a"]}, "p": {}}
    return dict(prev_map=prev, partitions_to_assign={"p": {}}, nodes_all=["a", "b"], nodes_to_remove=[], nodes_to_add=[],
                model={"primary": (0, 1), "replica": (1, 0)}, partition_weights={"h": 999999999})


def test_non_model_counts_above_int32_are_refused():
    lit = L.plan_next_map_ex(**wrapping_instance())
    assert lit["next_map"]["p"] == {"primary": ["b"]}          # what the device would miss with a wrapped count
    with pytest.raises(BlanceError, match=BOUND_MSG):
        _host.intern_plan(**wrapping_instance())


# ---- 2. literal oracle == array-form oracle at extreme values ------------------------------------------------------

PART_W = (-10**9, -7, -1, 0, 1, 999999999)
NODE_W = (-2**31, -1, 0, 1, 2, 2**30, 2**31 - 1)
STICK = (-5, 0, 2**31 - 1)


def extreme_instance(seed):
    """random_instance(seed)'s structure with extreme weights and stickiness drawn from a stream of its own.  Partition
    weights are cut back (the largest |w| first) until the instance is within the count bound."""
    kw = random_instance(seed)
    rnd = random.Random("value range %d" % seed)
    names = sorted(set(kw["prev_map"]) | set(kw["partitions_to_assign"] or ()))
    states = list(kw["model"])
    kw.pop("state_stickiness", None)
    if rnd.random() < 0.9:
        kw["partition_weights"] = {n: rnd.choice(PART_W) for n in names if rnd.random() < 0.7}
        if rnd.random() < 0.8:
            kw["state_stickiness"] = {s: rnd.choice(STICK) for s in states if rnd.random() < 0.8}
    else:
        kw.pop("partition_weights", None)
    if rnd.random() < 0.85:
        kw["node_weights"] = {n: rnd.choice(NODE_W) for n in kw["nodes_all"] if rnd.random() < 0.8}
        kw["booster"] = rnd.randint(0, 1)
    else:
        kw.pop("node_weights", None)
        kw.pop("booster", None)
    while True:
        try:
            return kw, _host.intern_plan(**copy.deepcopy(kw))
        except BlanceError as e:
            if BOUND_MSG not in str(e):
                raise
            w = kw["partition_weights"]
            w[max(w, key=lambda n: abs(w[n]))] = rnd.choice((-7, -1, 0, 1))


@pytest.mark.parametrize("chunk", range(20))
def test_literal_equals_fast_at_extreme_values(chunk):
    big = 0
    for seed in range(chunk * 100, (chunk + 1) * 100):
        kw, ip = extreme_instance(seed)
        big += any(abs(v) >= 10**9 - 1 for v in (kw.get("partition_weights") or {}).values())
        lit = L.plan_next_map_ex(**copy.deepcopy(kw))
        out = _host.plan_out(ip)
        assert FAST.oracle_fast_plan_next_map(ip.in_ptr, out.out_ptr) == 0
        next_map, warnings = _host.unintern_plan(ip, out)
        assert next_map == lit["next_map"], seed
        assert warnings == lit["warnings"], seed
        assert (out.iters_run, out.steps) == (lit["iterations"], lit["steps"]), seed
    assert big >= 3, big                       # partitions at +-10^9 survive the bound in some instances
