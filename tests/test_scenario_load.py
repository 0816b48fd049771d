"""blance_plan_scenarios_load with a NULL context, row by row, in the style of tests/test_wave_requests.py: one bad
argument at a time, each row pinning the exact (status, message) and how many schedule outputs the call cleared before
it failed.  Every row that passes its checks reaches the NULL context (CTX_FAN_OUT, as blance_plan_scenarios_exposure);
the exposure is optional here."""
import ctypes

import pytest

from test_wave_requests import INVALID, NULL_CTX, UNSUPPORTED, BAD_OPTS, BAD_SCEN, _Call

from blance_b200 import abi as api

NAME = "blance_plan_scenarios_load"


def _invoke(c, load=True):
    lib = api.capi()
    m = max(1, c.n) * max(1, c.nmc)
    c.load = (api.LoadOut * m)() if load else None
    return lib.blance_plan_scenarios_load(None, c.base_p, c.n, c.sc_p, c.opts, 0, 0, c.nmc, c.mc, None, c.out, c.sched,
                                          ctypes.byref(c.aopts), c.audit, c.eopts_p, c.series_cap, c.expo, c.load)


def _big(c):
    """n_parts x n_slots just over the load's static event bound, (n_slots + 1) x 2 x n_slots x n_parts < 2^31."""
    c.base.n_slots = 8
    c.base.n_parts = (1 << 31) // (9 * 2 * 8) + 1


# (row name, knobs, whether load is passed, an edit of the base, (status, message), schedule outputs cleared)
ROWS = [
    ("ok", {}, True, None, NULL_CTX, 4),
    ("no exposure", dict(expo=False), True, None, NULL_CTX, 4),
    ("no audit, no exposure", dict(audit=False, expo=False), True, None, NULL_CTX, 4),
    ("load", {}, False, None, (INVALID, NAME + ": load is NULL"), 4),
    ("n_move_conc", dict(nmc=0), True, None, (INVALID, NAME + ": the load needs a schedule: n_move_conc must be positive"), 0),
    ("sched", dict(sched=False), True, None,
     (INVALID, NAME + ": n_move_conc must be positive and move_conc and sched not NULL"), 0),
    ("base", dict(base=False), True, None, (INVALID, NAME + ": base is NULL"), 0),
    ("n", dict(n=0), True, None, (INVALID, NAME + ": n must be positive"), 0),
    ("out", dict(out=False), True, None, (INVALID, NAME + ": base, sc or out is NULL"), 0),
    ("scenario", BAD_SCEN, True, None, (INVALID, NAME + ": scenario 1: add_is_nil is neither 0 nor 1"), 4),
    ("opts", BAD_OPTS, True, None, (INVALID, NAME + ": scenario 1: opts.set has an unknown bit"), 4),
    ("series_cap", dict(series_cap=-1), True, None, (INVALID, NAME + ": series_cap is negative"), 4),
    ("events", dict(audit=False, expo=False), True, _big,
     (UNSUPPORTED, NAME + ": the load needs (n_slots + 1) x 2 x n_slots x n_parts < 2^31"), 4),
    # the load's checks come after the exposure's: a bad series_cap is reported before a NULL load
    ("series_cap and load", dict(series_cap=-1), False, None, (INVALID, NAME + ": series_cap is negative"), 4),
]


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_null_context_rows(row):
    _, knobs, load, edit, want, cleared = row
    c = _Call(False, **knobs)
    if edit:
        edit(c)
    st = _invoke(c, load)
    assert (st, api.capi().blance_last_error(None).decode()) == want
    assert c.cleared() == cleared


def test_declaration_matches_the_exposure_entry_plus_load():
    lib = api.capi()
    assert lib.blance_plan_scenarios_load.argtypes == lib.blance_plan_scenarios_exposure.argtypes + [ctypes.c_void_p]
