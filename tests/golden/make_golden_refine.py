"""
Generates tests/golden/peak_refine.npz by running the UNMODIFIED reference (AtomAI v0.8.1, CPU)
through oracle/ref_shim.py: atomai.utils.coords.peak_refinement on the normalised 1024 x 1024 golden
frame (tests/golden/bfo_1024.npz) with its 2410 Locator coordinates at d=None (and the d it chose),
d=3 and d=6; Locator(refine=True).run on a seeded three-frame synthetic stack; and a handful of
hand-placed atoms (.5 coordinates, windows on every border, a negative window start).  Run in the
build container only:

    python tests/golden/make_golden_refine.py

Inputs are rebuilt from the committed fixtures and seeds (refine_cases.py); only outputs are stored.
"""
import os
import sys
import time
import warnings
from collections import OrderedDict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import refine_cases as rc  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

aoi = import_reference()


def main():
    from atomai.predictors import Locator
    from atomai.utils.coords import get_nn_distances_, peak_refinement
    out = OrderedDict()
    frame, coords = rc.bfo_frame()
    for d in (None, 3, 6):
        t0 = time.time()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[f"bfo_d{d}"] = peak_refinement(frame, coords, d)
        print("bfo d", d, "%.1f s" % (time.time() - t0))
    out["bfo_default_d"] = np.int64(int(np.mean(np.concatenate(get_nn_distances_(coords)[0])) * 0.25))
    nn_out, stack = rc.locator_inputs()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loc = Locator(refine=True).run(nn_out, stack)
    unrefined = Locator(refine=False).run(nn_out)
    out["loc_keys"] = np.array(list(loc.keys()))
    for k, v in loc.items():
        out[f"loc_{k}"] = v
        out[f"loc_{k}_coords"] = unrefined[k]
        out[f"loc_{k}_d"] = np.int64(
            int(np.mean(np.concatenate(get_nn_distances_(unrefined[k])[0])) * 0.25))
        print("locator frame", k, len(v), "atoms, d =", int(out[f"loc_{k}_d"]))
    hand_img, hand_xy = rc.hand_case()
    out["hand"] = peak_refinement(hand_img, hand_xy, rc.HAND_D)
    np.savez_compressed(os.path.join(HERE, "peak_refine.npz"), **out)
    print("bytes", os.path.getsize(os.path.join(HERE, "peak_refine.npz")))


if __name__ == "__main__":
    main()
