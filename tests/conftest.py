"""pytest configuration: registers the `gpu` marker and makes the repo root and
oracle/ importable.  `-m "not gpu"` runs on the CPU-only builder; `-m gpu` runs
on an H100 and goes through the C ABI of libblance_b200.so."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")
