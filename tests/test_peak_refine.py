"""Peak refinement without a GPU: the scipy oracle against the goldens of the unmodified reference
(tests/golden/peak_refine.npz), the host side of atomai_b200's refinement (window rule, default d,
acceptance test, dict assembly) driven by the oracle's fits, the ABI's argument checks, and the
refine kernel's code in the built library."""
import ctypes
import os
import re
import shutil
import subprocess
import warnings

import numpy as np
import pytest

import golden_utils as gu
import refine_cases as rc
from atomai_b200 import _C
from atomai_b200.utils import coords
from oracle import refine_ref as ref


@pytest.fixture(scope="module")
def gold():
    return gu.load("peak_refine.npz")


def _quiet(fn, *a):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a)


@pytest.mark.parametrize("d", [None, 3, 6])
def test_oracle_matches_reference_bfo(gold, d):
    frame, xy = rc.bfo_frame()
    got = _quiet(ref.peak_refinement, frame, xy, d)
    assert np.array_equal(got, gold[f"bfo_d{d}"])
    assert ref.default_d(xy) == int(gold["bfo_default_d"]) == 4


def test_oracle_matches_reference_locator_and_hand(gold):
    _, stack = rc.locator_inputs()
    for k in gold["loc_keys"]:
        c = gold[f"loc_{k}_coords"]
        assert ref.default_d(c) == int(gold[f"loc_{k}_d"])
        assert np.array_equal(_quiet(ref.peak_refinement, stack[k, ..., 0], c), gold[f"loc_{k}"])
    img, xy = rc.hand_case()
    assert np.array_equal(ref.peak_refinement(img, xy, rc.HAND_D), gold["hand"])


def test_host_logic_with_oracle_fits(gold):
    """refine_frames with the scipy fits in place of the kernel reproduces the reference exactly:
    window origins (np.around half to even, numpy slice rules), per-frame default d, acceptance."""
    frame, xy = rc.bfo_frame()
    with pytest.warns(UserWarning, match="Defaulting to 1/4"):
        got = coords.refine_frames(frame[None], [xy], None, fit=ref.fit_table)[0]
    assert np.array_equal(got, gold["bfo_dNone"])
    _, stack = rc.locator_inputs()
    cs = [gold[f"loc_{k}_coords"] for k in gold["loc_keys"]]
    got = _quiet(coords.refine_frames, stack[..., 0], cs, None, ref.fit_table)
    for k, g in zip(gold["loc_keys"], got):
        assert np.array_equal(g, gold[f"loc_{k}"])
    img, hxy = rc.hand_case()
    got = coords.refine_frames(img[None], [hxy], rc.HAND_D, fit=ref.fit_table)[0]
    assert np.array_equal(got, gold["hand"])


def test_window_origins_follow_numpy_slicing():
    img = np.arange(40 * 36).reshape(40, 36)
    _, xy = rc.hand_case()
    for d in (1, 2, 4, 7):
        org = coords._window_origins(img.shape, xy, d)
        for c, o in zip(xy, org):
            win = ref.window(img, c, d)
            if win.shape == (2 * d, 2 * d):
                assert np.array_equal(win, img[o[0]:o[0] + 2 * d, o[1]:o[1] + 2 * d])
            else:
                assert (o == -1).all()
    org = coords._window_origins(img.shape, xy, 4)
    assert (org[:, 0] >= 0).sum() == 11 and list(org[10]) == [26, 8]   # the wrapped window


def test_refine_frames_rejects_out_of_range_d():
    xy = np.array([[10.0, 10.0, 0.0]])
    for d in (0, 17, -2):
        with pytest.raises(ValueError, match="1 <= d <= 16"):
            coords.refine_frames(np.zeros((1, 32, 32), np.float32), [xy], d, fit=ref.fit_table)
    out = coords.refine_frames(np.zeros((1, 32, 32), np.float32), [np.empty((0, 3))], None,
                               fit=ref.fit_table)
    assert out[0].shape == (0, 3)


def test_abi_rejects_bad_arguments_without_gpu():
    lib = _C.lib()
    p = ctypes.c_void_p(16)
    for d in (0, 17):
        assert lib.atomai_b200_peak_refine(p, 1, 32, 32, p, 1, d, p, p, None, None) != 0
        assert b"d=%d" % d in lib.atomai_b200_last_error()
    assert lib.atomai_b200_peak_refine(None, 1, 32, 32, p, 1, 4, p, p, None, None) != 0
    assert b"null" in lib.atomai_b200_last_error()
    assert lib.atomai_b200_peak_refine(p, 1, 32, 32, p, 1, 4, None, p, None, None) != 0
    assert lib.atomai_b200_peak_refine(p, 1, 32, 32, p, 1, 4, p, None, None, None) != 0
    assert lib.atomai_b200_peak_refine(p, 1, 32, 32, None, 1, 4, p, p, None, None) != 0


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_refine_kernel_is_sm_90a_and_spill_free():
    path = _C.build()
    sass = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True).stdout
    funcs = re.findall(r"Function : (\S+)", sass)
    assert any("peak_refine_kernel" in f for f in funcs)
    elf = subprocess.run([CUOBJDUMP, "-lelf", path], capture_output=True, text=True).stdout
    assert set(re.findall(r"sm_(\d+a?)", elf)) == {"90a"}
    res = subprocess.run([CUOBJDUMP, "-res-usage", path], capture_output=True, text=True).stdout
    lines = res.splitlines()
    i = next(i for i, l in enumerate(lines) if "peak_refine_kernel" in l and "Function" in l)
    m = re.search(r"REG:(\d+) STACK:(\d+)", lines[i + 1])
    # the only stack is the 40-byte buffer of the fp64 sin/cos large-argument reduction
    assert int(m.group(1)) <= 255 and int(m.group(2)) <= 40, m.group(0)
    sass_k = sass.split("peak_refine_kernel", 1)[1].split("Function :", 1)[0]
    assert "DMUL" in sass_k and "DADD" in sass_k      # the fits run in fp64
