"""
Generates tests/golden/blobs_ref.npz by running the UNMODIFIED reference's
atomai.utils.img.filter_cells_ and filter_cells (cv2.threshold, scipy.ndimage.label and
ndimage.sum) through oracle/ref_shim.py on the seeded cases of blobs_cases.py:

  <case>/out      the result (values, dtype and shape)
  <case>/error    the exception's first builtin base class, when the call raises

Run in the build container only:

    python tests/golden/make_golden_blobs.py
"""
import builtins
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import blobs_cases as bc  # noqa: E402


def error_name(e: BaseException) -> str:
    return next(t.__name__ for t in type(e).__mro__ if getattr(builtins, t.__name__, None) is t)


def main():
    from oracle import ref_shim
    ref = ref_shim.import_reference()
    from atomai.utils import img
    fns = {"filter_cells_": img.filter_cells_, "filter_cells": img.filter_cells}
    out = {}
    for name in bc.all_cases():
        try:
            res = bc.call(fns, name)
        except Exception as e:  # noqa: BLE001 — the exception type is the golden
            out[f"{name}/error"] = np.array(error_name(e))
            continue
        out[f"{name}/out"] = np.asarray(res)
    path = os.path.join(HERE, "blobs_ref.npz")
    np.savez_compressed(path, **out)
    print(f"{path}: {len(out)} arrays, {os.path.getsize(path)} bytes ({ref.__name__})")


if __name__ == "__main__":
    main()
