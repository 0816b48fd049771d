"""The raw C ABI of libblance_b200.so in ctypes (struct blance_plan_in / blance_plan_out of
include/blance_b200.h, the exported symbols, and the lazily loaded library handle).  Importing this module loads
NO native code - the table builders (synth.py, tables.py) and bench.py's CPU reference arm use it without
mapping the CUDA library; capi() loads the library on first use."""
import ctypes
import os

from . import build as _build


class BlanceError(RuntimeError):
    """A negative blance_status from the C ABI (the message is blance_last_error())."""


_I32_FIELDS = ("n_nodes", "n_node_ids", "n_states", "n_parts", "n_slots", "max_iters", "top_state", "booster_kind",
               "add_is_nil", "has_part_weights", "has_node_weights", "has_hier_rules")
_PTR_FIELDS = ("state_priority", "state_constraints", "state_slot_off", "state_stickiness", "state_has_stickiness",
               "node_removed", "node_added", "node_weight", "node_has_weight", "part_in_prev", "part_in_assign",
               "part_weight", "part_has_weight", "part_name_rank", "prev_rows", "prev_shape", "cur_rows", "cur_shape",
               "extra_tot_first", "extra_tot_rest")


class _PlanIn(ctypes.Structure):        # struct blance_plan_in, include/blance_b200.h
    _fields_ = ([(n, ctypes.c_int32) for n in _I32_FIELDS] + [(n, ctypes.c_void_p) for n in _PTR_FIELDS] +
                [("n_rules", ctypes.c_int32), ("n_hier_bits", ctypes.c_int32), ("rule_off", ctypes.c_void_p),
                 ("ie_mask", ctypes.c_void_p), ("engine", ctypes.c_int32)])


class _PlanOut(ctypes.Structure):
    _fields_ = [("next_rows", ctypes.c_void_p), ("next_shape", ctypes.c_void_p), ("warn", ctypes.c_void_p),
                ("iters_run", ctypes.c_int32), ("converged", ctypes.c_int32), ("steps", ctypes.c_int64),
                ("device_ms", ctypes.c_float), ("kernel_ms", ctypes.c_float), ("pass_ms", ctypes.c_float),
                ("sticky_steps", ctypes.c_int64)]


class _Scenario(ctypes.Structure):     # struct blance_scenario
    _fields_ = [("node_removed", ctypes.c_void_p), ("node_added", ctypes.c_void_p), ("add_is_nil", ctypes.c_int32),
                ("has_node_weights", ctypes.c_int32), ("node_weight", ctypes.c_void_p), ("node_has_weight", ctypes.c_void_p)]


class _ScenarioOut(ctypes.Structure):  # struct blance_scenario_out
    _fields_ = [("next_rows", ctypes.c_void_p), ("next_shape", ctypes.c_void_p), ("warn", ctypes.c_void_p),
                ("node_ops", ctypes.c_void_p), ("state_node_load", ctypes.c_void_p),
                ("iters_run", ctypes.c_int32), ("converged", ctypes.c_int32), ("steps", ctypes.c_int64),
                ("sticky_steps", ctypes.c_int64), ("parts_moved", ctypes.c_int64), ("ops_total", ctypes.c_int64),
                ("warn_parts", ctypes.c_int64)]


class _ScheduleOut(ctypes.Structure):  # struct blance_schedule_out
    _fields_ = [("rounds", ctypes.c_int32), ("moves_done", ctypes.c_int64), ("stuck_parts", ctypes.c_int64),
                ("max_batch", ctypes.c_int32), ("device_ms", ctypes.c_float)]


class _ScenarioScheduleOut(ctypes.Structure):  # struct blance_scenario_schedule_out
    _fields_ = [("rounds", ctypes.c_int32), ("moves_done", ctypes.c_int64), ("stuck_parts", ctypes.c_int64),
                ("max_batch", ctypes.c_int32), ("node_rounds", ctypes.c_void_p), ("node_last_round", ctypes.c_void_p),
                ("part_done_round", ctypes.c_void_p)]


class _ChainStage(ctypes.Structure):   # struct blance_chain_stage
    _fields_ = [("nodes", _Scenario), ("node_in_all", ctypes.c_void_p)]


class _ChainOut(ctypes.Structure):     # struct blance_chain_out
    _fields_ = [("node_ops", ctypes.c_void_p), ("ops_total", ctypes.c_int64), ("parts_moved", ctypes.c_int64)]


OPT_CONSTRAINTS, OPT_STICKINESS, OPT_PART_WEIGHTS, OPT_HIERARCHY = 1, 2, 4, 8   # enum blance_scenario_opt_set


class _ScenarioOpts(ctypes.Structure):  # struct blance_scenario_opts
    _fields_ = [("set", ctypes.c_uint32), ("state_constraints", ctypes.c_void_p), ("state_stickiness", ctypes.c_void_p),
                ("state_has_stickiness", ctypes.c_void_p), ("has_part_weights", ctypes.c_int32),
                ("n_weight_overrides", ctypes.c_int32), ("ow_part", ctypes.c_void_p), ("ow_weight", ctypes.c_void_p),
                ("ow_has", ctypes.c_void_p), ("extra_tot_first", ctypes.c_void_p), ("extra_tot_rest", ctypes.c_void_p),
                ("has_hier_rules", ctypes.c_int32), ("n_rules", ctypes.c_int32), ("n_hier_bits", ctypes.c_int32),
                ("rule_off", ctypes.c_void_p), ("ie_mask", ctypes.c_void_p)]


AUDIT_N2N = 1                                                                   # enum blance_audit_flags


class _AuditOpts(ctypes.Structure):    # struct blance_audit_opts
    _fields_ = [("flags", ctypes.c_uint32), ("n_domains", ctypes.c_int32), ("domain_parent", ctypes.c_void_p)]


class _AuditOut(ctypes.Structure):     # struct blance_audit_out
    _fields_ = [("short_slots", ctypes.c_void_p), ("over_slots", ctypes.c_void_p), ("rule_miss", ctypes.c_void_p),
                ("rule_tested", ctypes.c_void_p), ("dom_top", ctypes.c_void_p), ("dom_all", ctypes.c_void_p),
                ("dom_copies", ctypes.c_void_p), ("n2n", ctypes.c_void_p), ("part_flags", ctypes.c_void_p),
                ("short_parts", ctypes.c_int64), ("rule_miss_parts", ctypes.c_int64), ("no_top_parts", ctypes.c_int64),
                ("n2n_max", ctypes.c_int32), ("n2n_max_a", ctypes.c_int32), ("n2n_max_b", ctypes.c_int32),
                ("kernel_ms", ctypes.c_float)]


EXPO_METRICS = ("NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY", "COPIES")   # enum blance_expo_metric order


class _ExposureIn(ctypes.Structure):   # struct blance_exposure_in
    _fields_ = [("state_constraints", ctypes.c_void_p), ("top_state", ctypes.c_int32), ("n_domains", ctypes.c_int32),
                ("domain_parent", ctypes.c_void_p)]


class _ExposureOut(ctypes.Structure):  # struct blance_exposure_out
    _fields_ = [("rounds", ctypes.c_int32), ("series", ctypes.c_void_p), ("peak", ctypes.c_int64 * 6),
                ("peak_round", ctypes.c_int32 * 6), ("area", ctypes.c_int64 * 6), ("dom_peak", ctypes.c_void_p),
                ("dom_peak_round", ctypes.c_void_p), ("part_min_copies", ctypes.c_void_p), ("part_no_top", ctypes.c_void_p),
                ("part_flags", ctypes.c_void_p), ("kernel_ms", ctypes.c_float)]


_CAPI = None
EXPORTS = ("blance_ctx_create", "blance_ctx_create_multi", "blance_ctx_device_count", "blance_ctx_destroy", "blance_last_error", "blance_version", "blance_ctx_kernel_launches", "blance_plan_in_check", "blance_plan_next_map",
           "blance_plan_next_map_batch", "blance_plan_scenarios", "blance_plan_scenarios_ex", "blance_plan_scenarios_schedule", "blance_plan_scenarios_audit", "blance_plan_chains", "blance_map_audit", "blance_plan_audit", "blance_plan_upload", "blance_plan_run", "blance_plan_fetch", "blance_plan_free", "blance_plan_timing",
           "blance_calc_partition_moves", "blance_moves_create", "blance_moves_fetch", "blance_moves_available",
           "blance_moves_schedule", "blance_moves_schedule_fetch", "blance_moves_exposure", "blance_moves_free")


def capi():
    """ctypes handle of libblance_b200.so with argtypes set (the same symbols a cgo shim binds)."""
    global _CAPI
    if _CAPI is None:
        lib = ctypes.CDLL(os.environ.get("BLANCE_B200_LIB", _build.lib_path()))   # override: instrumented builds
        vp, i32 = ctypes.c_void_p, ctypes.c_int32
        lib.blance_ctx_create.argtypes = [ctypes.POINTER(vp), ctypes.c_int]
        lib.blance_ctx_create_multi.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_int), ctypes.c_int]
        lib.blance_ctx_device_count.argtypes = [vp]
        lib.blance_ctx_destroy.argtypes = [vp]
        lib.blance_ctx_destroy.restype = None
        lib.blance_last_error.argtypes = [vp]
        lib.blance_last_error.restype = ctypes.c_char_p
        lib.blance_ctx_kernel_launches.argtypes = [vp]
        lib.blance_ctx_kernel_launches.restype = ctypes.c_int64
        lib.blance_plan_in_check.argtypes = [vp, ctypes.c_char_p, i32]
        lib.blance_plan_next_map.argtypes = [vp, vp, vp]
        lib.blance_plan_next_map_batch.argtypes = [vp, i32, vp, vp]
        lib.blance_plan_scenarios.argtypes = [vp, vp, i32, vp, i32, i32, vp]
        lib.blance_plan_scenarios_ex.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp]
        lib.blance_plan_scenarios_schedule.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp]
        lib.blance_plan_scenarios_audit.argtypes = [vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        lib.blance_plan_chains.argtypes = [vp, vp, i32, i32, vp, vp, i32, i32, vp, vp]
        lib.blance_map_audit.argtypes = [vp, vp, vp, vp, vp, vp]
        lib.blance_plan_audit.argtypes = [vp, vp, vp, vp]
        lib.blance_plan_upload.argtypes = [vp, vp, ctypes.POINTER(vp)]
        lib.blance_plan_run.argtypes = [vp, vp]
        lib.blance_plan_fetch.argtypes = [vp, vp, vp]
        lib.blance_plan_timing.argtypes = [vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                                           ctypes.POINTER(ctypes.c_int32)]
        lib.blance_plan_free.argtypes = [vp, vp]
        lib.blance_plan_free.restype = None
        lib.blance_calc_partition_moves.argtypes = [vp, i32, i32, i32, vp, vp, vp, i32, i32, vp, vp, vp, vp]
        lib.blance_moves_create.argtypes = [vp, i32, i32, i32, vp, vp, vp, i32, i32, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_int64)]
        lib.blance_moves_fetch.argtypes = [vp, vp, vp, vp, vp, vp]
        lib.blance_moves_available.argtypes = [vp, vp, vp, vp, vp, vp]
        lib.blance_moves_schedule.argtypes = [vp, vp, i32, vp, vp]
        lib.blance_moves_schedule_fetch.argtypes = [vp, vp, vp, vp]
        lib.blance_moves_exposure.argtypes = [vp, vp, vp, vp]
        lib.blance_moves_free.argtypes = [vp, vp]
        lib.blance_moves_free.restype = None
        _CAPI = lib
    return _CAPI


PlanIn = _PlanIn
PlanOut = _PlanOut
Scenario = _Scenario
ScenarioOpts = _ScenarioOpts
ScenarioOut = _ScenarioOut
ScheduleOut = _ScheduleOut
ChainStage = _ChainStage
ChainOut = _ChainOut
ScenarioScheduleOut = _ScenarioScheduleOut
AuditOpts = _AuditOpts
AuditOut = _AuditOut
ExposureIn = _ExposureIn
ExposureOut = _ExposureOut
