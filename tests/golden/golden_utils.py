"""
Deterministic inputs / weights shared by make_golden.py (runs the unmodified reference in the build
container) and the parity tests (run anywhere).  Everything is derived from numpy's legacy
RandomState (MT19937, stable across numpy versions), so the goldens only store OUTPUTS.
"""
import os
from collections import OrderedDict

import numpy as np

GOLDEN_DIR = os.path.dirname(os.path.abspath(__file__))


def fill_state_dict(shapes: "OrderedDict[str, tuple]", seed: int) -> "OrderedDict[str, np.ndarray]":
    """Seeded, well-conditioned values for every entry of a reference state_dict.
    conv/linear weights ~ U(-a, a) with a = sqrt(3/fan_in); biases ~ U(-.1,.1);
    BN weight ~ U(.5,1.5) with random sign flips on 1/4 of the channels, BN bias ~ U(-.3,.3),
    running_mean ~ U(-.2,.2), running_var ~ U(.5,1.5), num_batches_tracked = 0."""
    rs = np.random.RandomState(seed)
    out = OrderedDict()
    bn_prefixes = {k.rsplit(".", 1)[0] for k in shapes if k.endswith("running_mean")}
    for k, shp in shapes.items():
        pre, leaf = k.rsplit(".", 1)
        if leaf == "num_batches_tracked":
            out[k] = np.zeros(shp, np.int64)
        elif pre in bn_prefixes:
            if leaf == "weight":
                w = rs.uniform(0.5, 1.5, shp)
                w *= np.where(rs.uniform(size=shp) < 0.25, -1.0, 1.0)
                out[k] = w.astype(np.float32)
            elif leaf == "bias":
                out[k] = rs.uniform(-0.3, 0.3, shp).astype(np.float32)
            elif leaf == "running_mean":
                out[k] = rs.uniform(-0.2, 0.2, shp).astype(np.float32)
            else:
                out[k] = rs.uniform(0.5, 1.5, shp).astype(np.float32)
        elif leaf == "weight":
            fan_in = int(np.prod(shp[1:])) if len(shp) > 1 else int(shp[0])
            a = (3.0 / max(fan_in, 1)) ** 0.5
            out[k] = rs.uniform(-a, a, shp).astype(np.float32)
        else:
            out[k] = rs.uniform(-0.1, 0.1, shp).astype(np.float32)
    return out


def images(seed: int, n: int, h: int, w: int) -> np.ndarray:
    """Synthetic 'atom lattice' images in [0,1]: Gaussian blobs on a jittered grid + noise."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = np.zeros((n, h, w), np.float32)
    for i in range(n):
        pitch = rs.uniform(5.0, 8.0)
        img = np.zeros((h, w), np.float32)
        for cy in np.arange(pitch / 2, h, pitch):
            for cx in np.arange(pitch / 2, w, pitch):
                jy, jx = rs.normal(0, 0.4, 2)
                img += np.exp(-((yy - cy - jy) ** 2 + (xx - cx - jx) ** 2) / (2 * 1.2 ** 2))
        img += rs.normal(0, 0.05, (h, w))
        img -= img.min()
        out[i] = img / (img.max() + 1e-6)
    return out


def labels(seed: int, n: int, h: int, w: int, nb_classes: int) -> np.ndarray:
    rs = np.random.RandomState(seed)
    lab = rs.randint(0, nb_classes, (n, h, w)).astype(np.int64)
    lab.reshape(n, -1)[:, :nb_classes] = np.arange(nb_classes)  # every class present
    return lab


def sample_flat(a: np.ndarray, stride: int = 97) -> np.ndarray:
    """Strided sample of a large tensor (keeps the fixture small but position-sensitive)."""
    return np.ascontiguousarray(a.reshape(-1)[::stride])


PART_BYTES = 900 * 1024   # every committed fixture file stays below 1 MB


class Arrays(OrderedDict):
    """np.load-like view (`files`, `[key]`) of a fixture stored as several part files."""
    @property
    def files(self):
        return list(self.keys())


def save(name: str, **arrays) -> None:
    """np.savez_compressed into GOLDEN_DIR; a fixture larger than PART_BYTES is written as
    <stem>.part<i>.npz files of at most PART_BYTES raw bytes each (an array larger than that is cut
    along axis 0 into '<key>@<j>' pieces, concatenated again by load())."""
    stem = name[:-len(".npz")]
    pieces = []
    for k, v in arrays.items():
        v = np.asarray(v)
        if v.nbytes <= PART_BYTES or v.ndim == 0:
            pieces.append((k, v))
        else:
            rows = max(1, PART_BYTES // max(1, v.nbytes // v.shape[0]))
            pieces += [(f"{k}@{j}", v[i:i + rows]) for j, i in enumerate(range(0, v.shape[0], rows))]
    if sum(v.nbytes for _, v in pieces) <= PART_BYTES:
        np.savez_compressed(os.path.join(GOLDEN_DIR, name), **dict(pieces))
        return
    parts, cur, size = [], {}, 0
    for k, v in pieces:
        if cur and size + v.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"{stem}.part{i}.npz"), **p)


def load(name: str):
    path = os.path.join(GOLDEN_DIR, name)
    if os.path.exists(path):
        return np.load(path, allow_pickle=False)
    stem, out, i = name[:-len(".npz")], Arrays(), 0
    pieces = OrderedDict()
    while os.path.exists(os.path.join(GOLDEN_DIR, f"{stem}.part{i}.npz")):
        with np.load(os.path.join(GOLDEN_DIR, f"{stem}.part{i}.npz"), allow_pickle=False) as z:
            for k in z.files:
                pieces.setdefault(k.split("@")[0], []).append(z[k])
        i += 1
    if not pieces:
        raise FileNotFoundError(path)
    for k, v in pieces.items():
        out[k] = v[0] if len(v) == 1 else np.concatenate(v, 0)
    return out


def subimage_inputs():
    """Seeded inputs of the sub-image extraction goldens: a (3, 40, 36, 2) float32 stack with a few
    NaNs, Locator-style coordinates {i: (N, 3)} with fractional, .5, edge and negative positions and
    two classes, one 2-D image and an (N, 2) coordinate array for it."""
    rs = np.random.RandomState(123)
    stack = rs.rand(3, 40, 36, 2).astype(np.float32)
    stack[1, 20, 20, 0] = np.nan
    stack[2, 5, 30, 1] = np.nan
    coords = {}
    for i in range(3):
        n = 60
        xy = np.concatenate([rs.rand(n, 1) * 46 - 3, rs.rand(n, 1) * 42 - 3], axis=1)
        xy[:6] = np.array([[3.5, 4.5], [2.5, 3.5], [0.0, 0.0], [39.0, 35.0], [-5.0, -6.0], [20.4, 20.6]])
        cls = (rs.rand(n, 1) > 0.7).astype(np.float64)
        coords[i] = np.concatenate([xy, cls], axis=1)
    single = rs.rand(33, 31)
    single_xy = np.concatenate([rs.rand(40, 1) * 33, rs.rand(40, 1) * 31], axis=1)
    return stack, coords, single, single_xy
