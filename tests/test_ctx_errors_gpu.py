"""A failing call reports its message on the context the caller passed: on a single-device context and on a
multi-device context, whose single-device entry points run on its first device (blance_ctx_create_multi([0])
works on a machine with one GPU)."""
import ctypes

import numpy as np
import pytest

from blance_b200 import tables

pytestmark = pytest.mark.gpu
INVALID_ARG = -1


@pytest.fixture(scope="module", params=["single", "multi"])
def ctx(request):
    c = tables.Context() if request.param == "single" else tables.Context(device_ids=[0])
    yield c
    c.close()


def assert_fails_with(ctx, st, text):
    assert st == INVALID_ARG
    assert text in ctx.lib.blance_last_error(ctx.ptr)


def tiny_moves(ctx):
    """One partition moving its single slot from node 0 to node 1."""
    return ctx.moves_create(np.array([0, 1]), np.array([[0]]), np.array([[1]]), False, 2)


def test_plan_upload_with_a_null_plan_in(ctx):
    plan = ctypes.c_void_p()
    assert_fails_with(ctx, ctx.lib.blance_plan_upload(ctx.ptr, None, ctypes.byref(plan)), b"plan_in is NULL")
    assert not plan.value


def test_plan_run_with_a_null_plan(ctx):
    assert_fails_with(ctx, ctx.lib.blance_plan_run(ctx.ptr, None), b"or plan is NULL")


def test_moves_create_with_a_null_out(ctx):
    slot_off = np.array([0, 1], np.int32)
    rows = np.array([0], np.int32)
    st = ctx.lib.blance_moves_create(ctx.ptr, 1, 1, 1, slot_off.ctypes.data, rows.ctypes.data, rows.ctypes.data, 0, 2, None, None)
    assert_fails_with(ctx, st, b"out is NULL")


def test_moves_schedule_fetch_without_a_schedule(ctx):
    handle, total_ops = tiny_moves(ctx)
    try:
        assert total_ops == 2
        assert_fails_with(ctx, ctx.lib.blance_moves_schedule_fetch(ctx.ptr, handle[0], None, None), b"no schedule")
        # the context and the handle still work after the failure
        round_off, sched_op, scalars = ctx.moves_schedule(handle, 1)
        assert scalars["moves_done"] == 2 and round_off[0] == 0 and round_off[-1] == 2
        assert sorted(sched_op) == [0, 1]
    finally:
        ctx.moves_free(handle)
