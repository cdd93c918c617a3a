"""
Seeded inputs of the utils.coords neighbour-search tests (tests/test_coords*.py,
tests/golden/make_golden_coords.py): jittered square lattices (8 px spacing) and movies of them,
image stacks to crop, and DBSCAN point sets with noise and with border points that touch two
clusters.  Coordinates are (x, y, class) rows in pixels; jitter keeps every distance tie-free.
"""
import numpy as np

SPACING = 8.0


def lattice(n: int, seed: int, jitter: float = 0.6, origin: float = 4.0, classes: int = 2,
            drop: float = 0.0) -> np.ndarray:
    """(n * n, 3) jittered square lattice rows (x, y, class), a fraction `drop` removed"""
    rng = np.random.default_rng(seed)
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    xy = origin + ij * SPACING + rng.normal(0, jitter, ij.shape)
    c = np.concatenate([xy, rng.integers(0, classes, (len(xy), 1)).astype(np.float64)], 1)
    if drop:
        c = c[rng.random(len(c)) >= drop]
    return c


def movie(frames: int, n: int, seed: int, jitter: float = 0.6, drift: float = 0.3,
          drop: float = 0.0) -> dict:
    """frames of one lattice whose atoms wander by `drift` px per frame"""
    rng = np.random.default_rng(seed)
    base = lattice(n, seed, jitter)
    out = {}
    for f in range(frames):
        c = base.copy()
        c[:, :2] += rng.normal(0, drift, (len(c), 2))
        if drop:
            c = c[rng.random(len(c)) >= drop]
        out[f] = c
    return out


def images(frames: int, h: int, w: int, seed: int, channels: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    shape = (frames, h, w) + ((channels,) if channels else ())
    return rng.random(shape).astype(np.float32)


def dbscan_points(seed: int = 0):
    """(rows, eps, min_samples): tight clusters over a movie, uniform noise, and two pairs of
    clusters joined only by a border point each (B listed before A, so the border point's lower
    cluster is B's)"""
    rng = np.random.default_rng(seed)
    mv = movie(12, 8, seed + 1, jitter=0.5, drift=0.15)
    pts = [mv[k] for k in range(12)]
    noise = np.concatenate([rng.uniform(0, 64, (40, 2)), np.zeros((40, 1))], 1)
    pts.append(noise)
    for x0 in (100.0, 120.0):
        b = np.array([[x0 + 0.95, 0], [x0 + 1.3, 0.2], [x0 + 1.3, -0.2], [x0 + 1.6, 0]])
        a = np.array([[x0 - 0.95, 0], [x0 - 1.3, 0.2], [x0 - 1.3, -0.2], [x0 - 1.6, 0]])
        x = np.array([[x0, 0.003]])
        for g in (x, b, a):
            g = g + rng.normal(0, 1e-3, g.shape)
            pts.append(np.concatenate([g, np.ones((len(g), 1))], 1))
    return np.concatenate(pts), 1.0, 4


def as_frames(rows: np.ndarray, n: int) -> dict:
    """rows split into n consecutive frames"""
    return {k: v for k, v in enumerate(np.array_split(rows, n))}
