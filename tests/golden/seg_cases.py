"""Seeded inputs of the segmentation-objective goldens (tests/golden/seg_objectives.npz), shared by
make_golden_seg.py and the tests: logits from numpy's legacy RandomState, labels from
golden_utils.labels.  No class probability comes closer than MARGIN to the 0.5 threshold, so the
thresholded class decisions do not depend on the last bits of the softmax / sigmoid."""
import numpy as np

import golden_utils as gu

MARGIN = 1e-3

# name -> (seed, N, C, H, W); C == 1 is the binary case ((N, 1, H, W) float labels)
CASES = {
    "mc3_32x48": (900, 2, 3, 32, 48),
    "mc3_24x37": (910, 2, 3, 24, 37),
    "mc5_16x20": (920, 2, 5, 16, 20),
    "bin_32x32": (930, 2, 1, 32, 32),
}

# three Adam steps (default Unet with dice, the 1-class nearest-upsampling Unet with focal): the
# seeds and shapes of the unet_default_3c / unet_nearest_1c goldens (tests/test_oracle.py CASES)
ADAM = {"dice": "unet_default_3c", "focal": "unet_nearest_1c"}


def _probs(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.float64)
    if x.shape[1] == 1:
        return 1.0 / (1.0 + np.exp(-x))
    e = np.exp(x - x.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def logits(seed: int, n: int, c: int, h: int, w: int) -> np.ndarray:
    rs = np.random.RandomState(seed)
    x = rs.normal(0.0, 2.0, (n, c, h, w)).astype(np.float32)
    while True:
        bad = (np.abs(_probs(x) - 0.5) < MARGIN).any(1)        # (n, h, w)
        if not bad.any():
            return x
        idx = np.nonzero(bad)
        x[idx[0], :, idx[1], idx[2]] = rs.normal(0.0, 2.0, (len(idx[0]), c)).astype(np.float32)


def labels(seed: int, n: int, c: int, h: int, w: int) -> np.ndarray:
    """(n, h, w) int64 class indices, or (n, 1, h, w) float32 binary masks for c == 1."""
    if c == 1:
        return (gu.labels(seed + 1, n, h, w, 2) > 0).astype(np.float32)[:, None]
    return gu.labels(seed + 1, n, h, w, c)


def case(name: str):
    seed, n, c, h, w = CASES[name]
    return logits(seed, n, c, h, w), labels(seed, n, c, h, w)
