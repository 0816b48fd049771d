"""The kernels the scenario exposure changed, read from the library's SASS (no device needed): the wave kernels keep
their reductions as REDs and gain no ATOMG, the exposure kernels stay free of ATOMG, and every kernel the change did not
touch is instruction-identical to the build before it (tests/golden/sass_digests_before_scenario_exposure.json)."""
import hashlib
import json
import os
import re
import subprocess

import pytest

from test_sass_guard import kernels  # noqa: F401  (the parsed SASS, a module-scoped fixture)


def _bodies(kernels, *names):  # noqa: F811
    out = {k: "\n".join(ls) for k, ls in kernels.items() if any(n in k for n in names)}
    assert out
    return out


def test_wave_kernels_reduce_with_red_and_never_atomg(kernels):  # noqa: F811
    bodies = _bodies(kernels, "k_wave_")
    for k, body in bodies.items():
        assert not re.search(r"ATOMG", body), k
    for name in ("k_wave_pick", "k_wave_first", "k_wave_node_ops"):
        assert any("REDG" in b for k, b in bodies.items() if name in k), name


# Kernels the exposure inside the wave changed on purpose: the exposure kernels (an instance dimension), k_wave_pick
# (records op rounds), k_wave_moves (records op states), and CUB's scan over the event counts, whose offsets are now
# 64-bit.  Every other kernel of the build before this change must be instruction-identical.
CHANGED = ("k_expo_", "k_wave_pick", "k_wave_moves", "DeviceScanKernelINS0_6detail4scan10policy_hubIxxxj")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sass_digests_before_scenario_exposure.json")


def _digest(lines):
    """sha256 of a kernel's instructions: encodings dropped, parameter-bank offsets masked (a grown struct argument
    shifts the offsets of the arguments after it without changing one instruction)."""
    ins = [re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][P]", re.sub(r"/\*.*?\*/", "", line).strip()) for line in lines]
    return hashlib.sha256("\n".join(ins).encode()).hexdigest()[:20]


def test_other_kernels_are_identical_to_the_build_before(kernels):  # noqa: F811
    golden = json.load(open(GOLDEN))
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    try:
        version = subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE, text=True, timeout=60).stdout
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("nvcc is not available")
    if golden["nvcc"] not in version:
        pytest.skip("the golden digests were taken with nvcc %s" % golden["nvcc"])
    kept = {k: d for k, d in golden["digests"].items() if not any(c in k for c in CHANGED)}
    assert len(kept) == len(golden["digests"]) - 11          # 7 exposure kernels, pick, moves and the two scan kernels
    bad = [k for k, d in kept.items() if k not in kernels or _digest(kernels[k]) != d]
    assert not bad, bad
