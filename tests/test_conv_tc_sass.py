"""Static checks of conv_tc_kernel with its two consumer warpgroups (no GPU): the stack frame of the
512-thread kernel stays within what the single-consumer kernel had, and ptxas did not serialise the
warpgroup MMAs (a serialised kernel waits for every HGMMA: one WARPGROUP.DEPBAR per HGMMA).
Skipped when the CUDA binary utilities are not installed."""
import os
import re
import shutil
import subprocess

import pytest

from atomai_b200 import _C

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
pytestmark = pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")


@pytest.fixture(scope="module")
def lib_path():
    return _C.build()


def test_conv_tc_stack_bound(lib_path):
    res = subprocess.run([CUOBJDUMP, "-res-usage", lib_path], capture_output=True, text=True).stdout
    lines = res.splitlines()
    found = False
    for i, line in enumerate(lines):
        if re.search(r"Function \S*conv_tc_kernel\S*:", line):
            m = re.search(r"REG:(\d+) STACK:(\d+)", lines[i + 1])
            assert m, lines[i + 1]
            assert int(m.group(1)) <= 128
            assert int(m.group(2)) <= 296, int(m.group(2))
            found = True
    assert found


def test_conv_tc_mmas_not_serialised(lib_path):
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", "conv_tc_kernel", lib_path],
                          capture_output=True, text=True).stdout
    if "HGMMA" not in sass:   # older cuobjdump without -fun matching: take the kernel's section
        full = subprocess.run([CUOBJDUMP, "-sass", lib_path], capture_output=True, text=True).stdout
        sass = next(b for b in re.split(r"\n\s*Function : ", full) if "conv_tc_kernel" in b.split("\n")[0])
    hgmma, depbar = sass.count("HGMMA"), sass.count("WARPGROUP.DEPBAR")
    assert hgmma >= 100
    assert depbar < hgmma, (hgmma, depbar)
