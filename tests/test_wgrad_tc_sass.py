"""Static checks of every wgrad_tc_kernel instantiation (no GPU): the register split between the
consumer and loader warpgroups (setmaxnreg) left no spills and no stack frame, and ptxas did not
serialise the warpgroup MMAs (a serialised kernel waits for every HGMMA: one WARPGROUP.DEPBAR per
HGMMA).  Skipped when the CUDA binary utilities are not installed."""
import os
import re
import shutil
import subprocess

import pytest

from atomai_b200 import _C

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")

# (N, kernel rows per unit, input channels on M) of every instantiation wgrad_plan can pick
INSTANTIATIONS = [(16, 3, True), (32, 3, True), (16, 3, False), (32, 3, False), (64, 3, False),
                  (16, 1, True), (32, 1, True), (16, 1, False), (32, 1, False), (64, 1, False)]


def _mangled(nb, th, trans):
    return f"wgrad_tc_kernelILi{nb}ELi{th}ELb{int(trans)}E"


@pytest.fixture(scope="module")
def lib_path():
    return _C.build()


@pytest.fixture(scope="module")
def sass_by_kernel(lib_path):
    full = subprocess.run([CUOBJDUMP, "-sass", lib_path], capture_output=True, text=True).stdout
    blocks = re.split(r"\n\s*Function : ", full)
    return {b.split("\n")[0]: b for b in blocks if "wgrad_tc_kernel" in b.split("\n")[0]}


@pytest.mark.parametrize("nb,th,trans", INSTANTIATIONS)
def test_wgrad_tc_no_spills_no_stack(lib_path, sass_by_kernel, nb, th, trans):
    res = subprocess.run([CUOBJDUMP, "-res-usage", lib_path], capture_output=True, text=True).stdout
    lines = res.splitlines()
    hits = [i for i, line in enumerate(lines) if _mangled(nb, th, trans) in line and "Function" in line]
    assert len(hits) == 1, hits
    m = re.search(r"STACK:(\d+)", lines[hits[0] + 1])
    assert m and int(m.group(1)) == 0, lines[hits[0] + 1]
    sass = next(b for name, b in sass_by_kernel.items() if _mangled(nb, th, trans) in name)
    assert not re.search(r"\bSTL(\.\w+)*\b", sass), "spill stores"


@pytest.mark.parametrize("nb,th,trans", INSTANTIATIONS)
def test_wgrad_tc_mmas_not_serialised(sass_by_kernel, nb, th, trans):
    sass = next(b for name, b in sass_by_kernel.items() if _mangled(nb, th, trans) in name)
    hgmma, depbar = sass.count("HGMMA"), sass.count("WARPGROUP.DEPBAR")
    assert hgmma >= 8 * th
    assert depbar < hgmma, (hgmma, depbar)
