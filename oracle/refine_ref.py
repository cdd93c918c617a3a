"""
CPU restatement of the reference's 2-D Gaussian peak refinement (atomai/utils/coords.py:86-231,
atomai/predictors/predictor.py:609-619) with scipy: the window rule, the per-frame default d, one
fit per atom and the acceptance test.  The Gaussian is evaluated in the reference's operation order
and the fit is the MINPACK lmdif call that scipy.optimize.curve_fit makes (leastsq on
f(x, *p) - y from the same start point), so on the CPU this reproduces the reference bit for bit
(tests/golden/peak_refine.npz).  `fit_window` also returns MINPACK's info code and nfev, which
curve_fit hides, for the per-fit comparisons against the GPU kernel.
"""
import warnings

import numpy as np
from scipy import optimize, spatial


def gaussian_2d(xy, amp, xo, yo, sigma_x, sigma_y, theta, offset):
    """Rotated 2-D Gaussian on the (x, y) grid, flattened (coords.py:152-176)."""
    x, y = xy
    cos2, sin2, sin2t = np.cos(theta) ** 2, np.sin(theta) ** 2, np.sin(2 * theta)
    a = cos2 / (2 * sigma_x ** 2) + sin2 / (2 * sigma_y ** 2)
    b = -sin2t / (4 * sigma_x ** 2) + sin2t / (4 * sigma_y ** 2)
    c = sin2 / (2 * sigma_x ** 2) + cos2 / (2 * sigma_y ** 2)
    dx, dy = x - xo, y - yo
    return (offset + amp * np.exp(-(a * (dx ** 2) + 2 * b * dx * dy + c * (dy ** 2)))).flatten()


def default_d(coordinates: np.ndarray) -> int:
    """int(1/4 of the mean distance to the two nearest neighbours)."""
    dist, _ = spatial.cKDTree(coordinates[:, :2]).query(coordinates[:, :2], k=3)
    dist = dist[~(dist == np.inf).any(1)]
    return int(np.mean(np.concatenate(dist[:, 1:])) * 0.25)


def fit_window(win: np.ndarray, d: int):
    """One fit of a (2d, 2d) window -> (popt (7,), MINPACK info, nfev)."""
    xy = np.mgrid[:win.shape[0], :win.shape[1]].astype(np.float64)
    ydata = win.flatten().astype(np.float64)
    p0 = np.array((win[d, d], d, d, 1, 1, 0, 0), np.float64)
    popt, _, infodict, _, ier = optimize.leastsq(
        lambda p: gaussian_2d(xy, *p) - ydata, p0, full_output=True)
    return popt, int(ier), int(infodict["nfev"])


def window(img: np.ndarray, c: np.ndarray, d: int):
    cx, cy = int(np.around(c[0])), int(np.around(c[1]))
    return img[cx - d:cx + d, cy - d:cy + d]


def peak_refinement(img: np.ndarray, coordinates: np.ndarray, d=None) -> np.ndarray:
    """Refined (N, 3) coordinates of one frame (coords.py:179-231)."""
    if d is None:
        warnings.warn("The d-value for bounding box not found. "
                      "Defaulting to 1/4 of mean atomic distance.", stacklevel=2)
        d = default_d(coordinates)
    out = []
    for c in coordinates[:, :2]:
        xyc = c
        win = window(img, c, d)
        if win.shape == (2 * d, 2 * d):
            if not np.isfinite(win).all():
                raise ValueError("array must not contain infs or NaNs")
            popt, info, _ = fit_window(win, d)
            if 1 <= info <= 4 and np.linalg.norm(popt[1:3] - d) < 3:
                xyc = popt[1:3] + np.around(c) - d
        out.append(xyc)
    return np.concatenate((np.array(out), coordinates[:, 2:3]), axis=-1)


def fit_table(stack: np.ndarray, table: np.ndarray, dmax: int):
    """The fits of a (K, 4) table {frame, row0, col0, d} over an (n, H, W) stack, as the native
    launch returns them: popt (K, 7), info (K,)."""
    popt = np.empty((len(table), 7))
    info = np.empty(len(table), np.int32)
    for k, (f, r0, c0, d) in enumerate(np.asarray(table, np.int64)):
        assert 1 <= d <= dmax
        win = np.asarray(stack[f])[r0:r0 + 2 * d, c0:c0 + 2 * d]
        popt[k], info[k], _ = fit_window(win, int(d))
    return popt, info
