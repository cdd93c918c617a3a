"""
Inputs of the peak-refinement goldens (make_golden_refine.py) and of their parity tests, rebuilt from
committed fixtures and seeds.
"""
import numpy as np

import golden_utils as gu

HAND_D = 4


def normalise(img: np.ndarray) -> np.ndarray:
    """The min-max normalisation SegPredictor applies (torch_format_image), as float32."""
    img = img[None, None]
    return ((img - img.min()) / np.ptp(img)).astype(np.float32)[0, 0]


def bfo_frame():
    """The 1024 x 1024 golden frame as the Locator sees it, and its 2410 Locator coordinates."""
    g = gu.load("bfo_1024.npz")
    return normalise(g["image"]), np.asarray(g["coordinates"], np.float64)


def locator_inputs():
    """A (3, 192, 192, 2) 'network output' and the (3, 192, 192, 1) image stack it came from:
    seeded lattices upsampled 3x (cubic spline) so that each frame's default d is 3 or more."""
    from scipy import ndimage
    imgs = ndimage.zoom(gu.images(31, 3, 64, 64), (1, 3, 3), order=3)
    imgs = (imgs - imgs.min()) / np.ptp(imgs)
    nn_out = np.stack([imgs, 1 - imgs], axis=-1).astype(np.float32)
    return nn_out, imgs[..., None].astype(np.float32)


def hand_case():
    """A 40 x 36 crop of the golden frame and hand-placed atoms for d = 4: .5 coordinates (np.around
    rounds half to even), windows touching each border, windows cut by a border, and starts below
    zero (numpy wraps them, usually to an empty slice, once to a full window)."""
    frame, _ = bfo_frame()
    img = np.ascontiguousarray(frame[300:340, 400:436])
    xy = np.array([
        [4.0, 4.0], [35.5, 31.5], [3.5, 10.5], [4.5, 27.5], [19.5, 16.5], [18.5, 17.5],
        [20.5, 4.0], [36.0, 20.0], [12.0, 32.0], [2.5, 20.0], [-10.0, 12.0], [-40.0, 5.0],
        [37.0, 20.0], [20.5, 33.0], [22.49, 9.51], [15.0, -3.0],
    ])
    cls = (np.arange(len(xy)) % 3)[:, None].astype(np.float64)
    return img, np.concatenate([xy, cls], axis=1)
