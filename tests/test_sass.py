"""Static checks of the built library (no GPU): the hot kernels really are wgmma / TMA code for
sm_90a (SASS opcodes), the thin-channel kernels and the weight-gradient kernel do not spill, and
the convolution kernel fits its 512-thread CTA (<= 128 registers at launch) with a bounded stack.
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


def _per_kernel(text, header):
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(header, line)
        if m:
            cur = out.setdefault(m.group(1), [])
        elif cur is not None:
            cur.append(line)
    return out


def test_only_sm_90a_code(lib_path):
    elf = subprocess.run([CUOBJDUMP, "-lelf", lib_path], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", elf))
    assert archs == {"90a"}, archs


def test_tensor_core_kernels_carry_wgmma_tma(lib_path):
    sass = subprocess.run([CUOBJDUMP, "-sass", lib_path], capture_output=True, text=True).stdout
    k = _per_kernel(sass, r"Function : (\S+)")
    conv = "\n".join(next(v for n, v in k.items() if "conv_tc_kernel" in n))
    wgrad = "\n".join(next(v for n, v in k.items() if "wgrad_tc_kernel" in n))
    for op in ("HGMMA", "UTMALDG", "UBLKCP", "USETMAXREG", "SYNCS"):
        assert op in conv, f"conv_tc_kernel lacks {op}"
    assert "HGMMA" in wgrad, "wgrad_tc_kernel lacks HGMMA"
    assert conv.count("HGMMA") >= 100 and wgrad.count("HGMMA") >= 8
    assert "HMMA.16816" not in conv and "HMMA.1688" not in conv      # no legacy mma.sync path


def test_registers_and_stack(lib_path):
    res = subprocess.run([CUOBJDUMP, "-res-usage", lib_path], capture_output=True, text=True).stdout
    usage = {}
    name = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            usage[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    assert usage, "no resource usage parsed"
    for n, (reg, stack) in usage.items():
        if "conv_tc_kernel" in n:
            assert reg <= 128, (n, reg)          # 512 threads x 128 = the whole register file
            assert stack <= 384, (n, stack)      # epilogue temporaries spilled today; must not grow
        if "wgrad_tc_kernel" in n:
            assert stack == 0, (n, stack)        # accumulators and staged operands stay in registers
        # the BatchNorm-backward and max-pool-backward bodies at both widths (W = 4 and 1, every
        # pool_bwd STATS variant); the digit is the mangled name's length, which keeps avgpool out
        if any(t in n for t in ("_tile_kernel", "_quad_kernel", "adam_multi")) or re.search(
                r"\d(bn_lrelu_bwd|bn_bwd_reduce|pool_bwd)_kernelILi[14]E", n):
            assert stack == 0, (n, stack)        # streaming kernels: nothing spilled
