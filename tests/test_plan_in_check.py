"""blance_plan_in_check (include/blance_b200.h): the content check of one instance's tables.  Host code only - no
device, no compute: every table the other tests feed to the planner (the reference's golden cases and the random
instances through the interning layer, the synthetic configurations) must pass, and each documented invariant must
be caught when it is broken.  CPU only."""
import ctypes

import numpy as np
import pytest

import golden_util as G
from randgen import random_instance

from blance_b200 import _host, abi, synth

OK, INVALID, UNSUPPORTED = 0, -1, -2


def check_ptr(in_ptr):
    msg = ctypes.create_string_buffer(256)
    st = abi.capi().blance_plan_in_check(in_ptr, msg, 256)
    return st, msg.value.decode()


def check_tables(t):
    s = t.struct()
    return check_ptr(ctypes.addressof(s))


@pytest.mark.parametrize("c", G.plan_cases(), ids=G.case_id)
def test_golden_cases_pass(c):
    ip = _host.intern_plan(**G.plan_kwargs(c))
    assert check_ptr(ip.in_ptr) == (OK, "")


def test_random_instances_pass():
    for seed in range(600):
        ip = _host.intern_plan(**random_instance(seed))
        assert check_ptr(ip.in_ptr) == (OK, ""), seed


@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
def test_synthetic_configurations_pass(cfg):
    P = {1: None, 2: 512, 3: 1024, 4: 2048, 5: 256}[cfg]
    assert check_tables(synth.make_fresh(cfg, P=P)) == (OK, "")
    if cfg == 4:
        assert check_tables(synth.make_rebalance(4, P=P)) == (OK, "")
        assert check_tables(synth.make_rebalance(4, P=1024, N=1500)) == (OK, "")


def broken(mutate):
    t = synth.make_rebalance(4, P=256, N=96)
    mutate(t)
    return check_tables(t)


def test_each_invariant_is_caught():
    def set_(name, idx, val):
        def f(t):
            a = getattr(t, name).copy()
            a[idx] = val
            setattr(t, name, a)
        return f

    st, why = broken(set_("prev_rows", (7, 1), 96 + 1000))
    assert st == INVALID and "prev_rows" in why
    st, why = broken(set_("cur_rows", (0, 0), -2))
    assert st == INVALID and "cur_rows" in why
    st, why = broken(set_("state_slot_off", 0, 1))           # (also shrinks state 0's range: either message is right)
    assert st == INVALID and why
    st, why = broken(set_("cur_shape", (3, 1), 3))
    assert st == INVALID and "cur_shape" in why
    st, why = broken(set_("part_name_rank", 5, 4))
    assert st == INVALID and "twice" in why
    st, why = broken(set_("part_name_rank", 5, -1))
    assert st == INVALID and "part_name_rank" in why
    st, why = broken(set_("part_name_rank", 5, 1 << 30))
    assert st == INVALID and "part_name_rank" in why
    # ranks above n_parts are legal as long as they are unique
    assert broken(set_("part_name_rank", 5, 1 << 20))[0] == OK

    def gap(t):                                # replica slots are 1 and 2 of every row: empty the first one only
        a = t.prev_rows.copy()
        assert a[9, 2] >= 0
        a[9, 1] = -1
        t.prev_rows = a
    st, why = broken(gap)
    assert st == INVALID and "after an empty slot" in why

    def heavy(t):
        w = t.part_weight.copy(); h = t.part_has_weight.copy()
        w[11] = 1_000_000_000; h[11] = 1
        t.part_weight, t.part_has_weight, t.has_part_weights = w, h, 1
    st, why = broken(heavy)
    assert st == UNSUPPORTED and "999999999" in why


@pytest.mark.parametrize("k,n_rules,ok", [(8, 4, True), (16, 2, True), (11, 3, False), (1, 33, False)])
def test_hierarchy_picks_per_step_at_most_32(k, n_rules, ok):
    """rules x constraints of one state is the number of hierarchy picks a step makes: 32 fit, 33 are rejected."""
    t = synth.PlanTables(64, 1, 16, [0], [k])
    t.has_hier_rules = 1
    t.rule_off, mask = synth.hierarchy_masks(64, (8, 8), {0: [(2, 1)] * n_rules}, 1)
    t.n_rules = mask.shape[0]
    t.ie_mask = mask.reshape(-1)
    st, why = check_tables(t)
    if ok:
        assert (st, why) == (OK, "")
    else:
        assert st == UNSUPPORTED and "rules x constraints" in why


def test_structure_errors_come_first_and_null_is_safe():
    assert abi.capi().blance_plan_in_check(None, None, 0) == INVALID
    t = synth.make_fresh(1)
    t.n_states = 9                             # more than 8 model states
    st, why = check_tables(t)
    assert st in (INVALID, UNSUPPORTED) and why
