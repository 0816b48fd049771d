"""What the compiled library must (not) contain - read from its SASS with cuobjdump, no device needed.

* no value-less atomic compiled WITH a return value (`ATOMG ... PT, RZ`): the pass kernels' atomicAdd calls whose
  result nobody reads were emitted that way, and the speculative kernel's leader then waited for an L2 round trip at
  its next branch.  They go through red_add()
  (pass_common.cuh) now; this guards the next edit.
* the speculative pass kernel is fed by TMA bulk copies completing on an mbarrier (UBLKCP / SYNCS) and reduces
  with redux.sync (REDUX): the sm_90a instructions DESIGN.md section 3 describes are really in the binary."""
import re
import shutil
import subprocess

import pytest

from blance_b200 import build

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def kernels():
    try:
        txt = subprocess.run([CUOBJDUMP, "-sass", build.lib_path()], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300).stdout
    except (OSError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump is not available")
    if "Function :" not in txt:
        pytest.skip("cuobjdump printed no SASS")
    out, name = {}, None
    for line in txt.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,6}\*/", line):
            out[name].append(line)
    return out


def test_no_atomic_with_a_discarded_return_value_in_the_pass_kernels(kernels):
    bad = [(k, l.strip()[:90]) for k, ls in kernels.items() if "k_assign_pass" in k for l in ls if re.search(r"ATOMG\.\S+ PT, RZ,", l)]
    assert not bad, bad[:5]


def test_speculative_pass_kernel_uses_tma_mbarrier_redux_and_red(kernels):
    spec = {k: ls for k, ls in kernels.items() if "k_assign_pass_spec" in k}
    assert len(spec) == 4                                  # K = 1 .. 4
    for k, ls in spec.items():
        body = "\n".join(ls)
        for op in ("UBLKCP", "SYNCS", "REDUX", "REDG"):
            assert op in body, (k, op)
