"""
Host restatement of the lattice masks of atomai/utils/imgen.py:82-229, for sizes beyond the
goldens: one numpy slice assignment per atom in input order (so the last atom wins), with the
mask template made once per class.  The caller's coordinates are not modified.
"""
import numpy as np


def _stamp(out, x: int, y: int, t: np.ndarray) -> None:
    r1, r2 = int(t.shape[0] / 2 + .5), int(t.shape[0] / 2 - .5)
    out[x - r1:x + r2, y - r1:y + r2] = t


def lattice_mask(lattice: np.ndarray, xy: np.ndarray, make_mask, scale: int = 7,
                 rmask: int = 5) -> np.ndarray:
    out = np.zeros_like(lattice)
    if len(xy):
        _, t = make_mask(scale, rmask)
        for x, y in np.around(np.asarray(xy, np.float64)).astype(np.int64):
            _stamp(out, x, y, t)
    return out


def multiclass_mask(shape, xyz: np.ndarray, make_mask, scale: int = 7,
                    rmask: int = 7) -> np.ndarray:
    z = xyz[:, -1] + (1 if (xyz[:, -1] == 0).any() else 0)
    classes = np.unique(z)
    out = np.zeros((shape[0], shape[1], len(classes)))
    templates = [make_mask(scale, rmask, c)[1] for c in classes]
    for (x, y), c in zip(np.around(xyz[:, :2]).astype(np.int64), np.searchsorted(classes, z)):
        _stamp(out[..., c], x, y, templates[c])
    out = np.concatenate([out, (1 - out.sum(-1))[..., None]], -1)
    out[out < 0] = 0
    return out
