"""
Cases of the Regressor / Classifier goldens (make_golden_regcls.py) and their deterministic
inputs and weights, shared by the generator and the tests.  Weights come from
golden_utils.fill_state_dict on the reference's state_dict shapes; large arrays are stored as
golden_utils.sample_flat samples.
"""
from collections import OrderedDict

import numpy as np

import golden_utils as gu

# kind, output size (out_dim / nb_classes), input channels, batch, image side, seed
CASES = OrderedDict([
    ("reg_64", dict(kind="reg", out=2, ic=1, n=8, hw=64, seed=11)),      # ends at 2 x 2
    ("cls_100", dict(kind="cls", out=4, ic=1, n=4, hw=100, seed=12)),    # odd sizes: 50 25 13 7 4
    ("reg3_32", dict(kind="reg", out=2, ic=3, n=8, hw=32, seed=13)),     # 3 channels, ends at 1 x 1
])
ADAM_STEPS = 3
PREDICT = dict(n=6, hw=64, seed=21)


def sampled(a: np.ndarray) -> np.ndarray:
    return gu.sample_flat(np.asarray(a), 97)


def inputs(c):
    """(x (n, ic, hw, hw) float32, y): float32 (n, out) targets or int64 (n,) labels."""
    x = np.stack([gu.images(c["seed"] + 100 * k, c["n"], c["hw"], c["hw"]) for k in range(c["ic"])],
                 axis=1)
    rs = np.random.RandomState(c["seed"])
    if c["kind"] == "reg":
        y = rs.normal(0, 1, (c["n"], c["out"])).astype(np.float32)
    else:
        y = (np.arange(c["n"]) % c["out"]).astype(np.int64)
        rs.shuffle(y)
    return np.ascontiguousarray(x, np.float32), y


def weights(shapes, c):
    return gu.fill_state_dict(shapes, c["seed"])
