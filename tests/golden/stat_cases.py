"""Seeded inputs of the stat goldens (tests/golden/make_golden_stat.py) and of the stat tests:
the goldens store outputs only, both sides regenerate the inputs from these functions."""
import numpy as np

# (window, channels, frames): movies of atoms whose neighbourhoods take one of three patterns
SEPARATED = {"w7c1": (7, 1, 1), "w16c3": (16, 3, 1), "w32c3": (32, 3, 6)}
OVERLAP = {"n2000d50k5": (2000, 50, 5, 3), "n1500d49k3": (1500, 49, 3, 11)}   # (N, d, K, seed)


def separated_movie(window, channels, frames, seed=0, grid=6):
    """(frames, H, W, channels) float32 images and Locator-style coordinates {frame: (n, 3)}:
    a grid of atoms (class 0) plus decoys (class 1); each atom's window shows one of three
    well-separated patterns, which changes between frames for a third of the atoms."""
    rs = np.random.RandomState(seed)
    step = window + 4
    H = W = grid * step + window
    n = grid * grid
    centres = np.array([(window // 2 + 2 + i * step, window // 2 + 2 + j * step)
                        for i in range(grid) for j in range(grid)], dtype=np.float64)
    yy, xx = np.mgrid[:window, :window] - (window - 1) / 2.0
    rr = np.sqrt(yy ** 2 + xx ** 2) / window
    patterns = [np.exp(-(rr / 0.15) ** 2), np.exp(-((rr - 0.35) / 0.08) ** 2),
                (np.abs(yy) < window / 6) * 1.0]
    kind = rs.randint(0, 3, n)
    imgs = np.zeros((frames, H, W, channels), np.float32)
    coords = {}
    for f in range(frames):
        if f:
            flip = rs.rand(n) < 0.33
            kind = np.where(flip, rs.randint(0, 3, n), kind)
        for a, (cx, cy) in enumerate(centres):
            x0, y0 = int(cx) - window // 2, int(cy) - window // 2
            for c in range(channels):
                imgs[f, x0:x0 + window, y0:y0 + window, c] = \
                    (1.0 + 0.3 * c) * patterns[kind[a]] + 0.02 * rs.randn(window, window)
        jitter = 0.2 * rs.randn(n, 2)
        decoys = np.array([[3.0, 3.0, 1.0], [H - 4.0, W - 4.0, 1.0]])
        coords[f] = np.concatenate(
            [np.concatenate([centres + jitter, np.zeros((n, 1))], 1), decoys], 0)
    return imgs, coords


def overlapping(N, d, K, seed):
    """(N, d) float32 mixture of K Gaussians with diagonal covariances that overlap."""
    rs = np.random.RandomState(seed)
    means = rs.randn(K, d) * 0.2
    scales = 0.5 + rs.rand(K, d)
    lab = rs.randint(0, K, N)
    return (means[lab] + scales[lab] * rs.randn(N, d)).astype(np.float32)


def lloyd_init(X, K, seed):
    """K distinct rows of X as an initial centre array."""
    rs = np.random.RandomState(seed)
    return X[rs.choice(len(X), K, replace=False)].copy()
