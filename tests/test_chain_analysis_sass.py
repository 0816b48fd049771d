"""The kernel blance_plan_chains_exposure added, read from the library's SASS (no device needed): k_chain_fold owns
every element it writes, so it has no ATOMG, and every kernel of the build before it is instruction-identical
(tests/golden/sass_digests_before_chain_analysis.json).  The node-load kernels and their CUB instantiations, added
after it, are pinned the same way (tests/golden/sass_digests_load.json)."""
import json
import os
import subprocess

import pytest

from test_sass_guard import kernels  # noqa: F401  (the parsed SASS, a module-scoped fixture)
from test_scenario_exposure_sass import _digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sass_digests_before_chain_analysis.json")
LOAD_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sass_digests_load.json")


def test_chain_fold_has_no_atomics(kernels):  # noqa: F811
    fold = [k for k in kernels if "k_chain_fold" in k]
    assert len(fold) == 1
    body = "\n".join(kernels[fold[0]])
    assert "ATOMG" not in body and "REDG" not in body


def test_every_kernel_is_identical_to_its_golden_digest(kernels):  # noqa: F811
    golden, load = json.load(open(GOLDEN)), json.load(open(LOAD_GOLDEN))
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    try:
        version = subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE, text=True, timeout=60).stdout
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("nvcc is not available")
    if golden["nvcc"] not in version or load["nvcc"] not in version:
        pytest.skip("the golden digests were taken with nvcc %s" % golden["nvcc"])
    want = dict(golden["digests"], **load["digests"])
    assert all(golden["digests"][k] == d for k, d in load["digests"].items() if k in golden["digests"])
    bad = [k for k, d in want.items() if k not in kernels or _digest(kernels[k]) != d]
    assert not bad, bad
    assert set(kernels) - set(want) == {k for k in kernels if "k_chain_fold" in k}
