"""
Generates tests/golden/gp_input.npz by running the UNMODIFIED reference (AtomAI v0.8.1, CPU)
through oracle/ref_shim.py: atomai.utils.prepare_gp_input and get_lengthscale_constraints on small
seeded sparse images (odd, square, non-square, a single row, one 3-D stack).  Run in the build
container only:

    python tests/golden/make_golden_gpr.py

The input images are stored next to the outputs.
"""
import os
import sys
from collections import OrderedDict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.ref_shim import import_reference  # noqa: E402

aoi = import_reference()

SHAPES = {"5x7": (5, 7), "8x8": (8, 8), "9x4": (9, 4), "1x6": (1, 6), "3x4x5": (3, 4, 5)}


def sparse_image(shape, seed, keep=0.3):
    rs = np.random.RandomState(seed)
    img = (rs.rand(*shape) + 0.1).astype(np.float32)
    return img * (rs.rand(*shape) < keep)


def main():
    from atomai.utils import get_lengthscale_constraints, prepare_gp_input
    out = OrderedDict()
    for i, (tag, shape) in enumerate(SHAPES.items()):
        img = sparse_image(shape, 40 + i)
        x, y, full = prepare_gp_input(img)
        lo, hi = get_lengthscale_constraints(full)
        out[f"{tag}/image"] = img
        out[f"{tag}/x"], out[f"{tag}/y"], out[f"{tag}/full"] = x, y, full
        out[f"{tag}/lower"], out[f"{tag}/upper"] = np.array(lo), np.array(hi)
        print(tag, x.shape, full.shape, lo, hi)
    np.savez_compressed(os.path.join(HERE, "gp_input.npz"), **out)


if __name__ == "__main__":
    main()
