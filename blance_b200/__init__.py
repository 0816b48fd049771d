"""blance_b200 — an H100-native (sm_90a) drop-in for the hot path of couchbase/blance:
PlanNextMapEx (api.go:147-157; plan.go:23-331) and CalcPartitionMoves (moves.go:41-119).

The product is the C-ABI library `blance_b200/lib/libblance_b200.so`
(include/blance_b200.h) plus the C++ host mirror of blance's api.go
(blance_b200/csrc/host_api.hpp).  This Python package is only a thin face over
that host mirror so tests and bench.py can call it with dicts; names follow the
reference (PlanNextMapEx, PlanNextMap, CalcPartitionMoves, ...).

There is no CPU fallback: importing works anywhere the shared objects were built,
but every compute call raises BlanceError without a CUDA device.
"""
import importlib
import os

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))

_API_NAMES = ("AuditMap", "BOOSTER_CBGT_MAX", "BOOSTER_NONE", "BlanceError", "CalcPartitionMoves", "CalcPartitionMovesMap",
              "NodeStateOp", "OrchestrateExposure", "OrchestrateSchedule", "OrchestratorOptions", "PlanNextMap", "PlanNextMapEx", "PlanNextMapOptions",
              "PlanNextMapChains", "PlanNextMapScenarios", "capi")
__all__ = ["AuditMap", "PlanNextMap", "PlanNextMapEx", "PlanNextMapOptions", "PlanNextMapScenarios", "PlanNextMapChains", "CalcPartitionMoves", "CalcPartitionMovesMap",
           "NodeStateOp", "OrchestrateExposure", "OrchestrateSchedule", "OrchestratorOptions", "BlanceError", "BOOSTER_NONE", "BOOSTER_CBGT_MAX", "capi"]


def __getattr__(name):
    """The native pieces (_host*.so, libblance_b200.so) load on first use of the API, not at import: the table
    builders `blance_b200.synth` / `blance_b200.tables` stay importable by processes that must not map the
    product's libraries (bench.py's CPU reference arm)."""
    if name == "_host" or name == "api" or name in _API_NAMES:
        if not (os.path.exists(_build.lib_path()) and os.path.exists(_build.host_module_path())):
            _build.build_all()
        mod = importlib.import_module("." + ("_host" if name == "_host" else "api"), __name__)
        return mod if name in ("_host", "api") else getattr(mod, name)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
