"""Loads the CPU oracles (oracle/ — TEST INFRASTRUCTURE).  Builds them on demand
with oracle/Makefile when the shared objects are missing (they are git-ignored
build products that __graft_entry__.build() normally leaves in oracle/)."""
import glob
import importlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")


def _build():
    subprocess.run(["make", "-s", "-C", ORACLE, "all"], check=True)


def literal():
    """The pybind11 module of the literal C++ oracle (oracle/literal.cpp)."""
    if not glob.glob(os.path.join(ORACLE, "_literal*.so")):
        _build()
    if ORACLE not in sys.path:
        sys.path.insert(0, ORACLE)
    return importlib.import_module("_literal")


def fast_lib_path():
    path = os.path.join(ORACLE, "libfast_oracle.so")
    if not os.path.exists(path):
        _build()
    return path
