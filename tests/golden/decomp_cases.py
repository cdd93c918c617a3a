"""Seeded inputs of the decomposition goldens (tests/golden/make_golden_decomp.py) and of the
decomposition tests: the goldens store outputs only, both sides regenerate the inputs here."""
import numpy as np

import stat_cases

PCA = {"gauss_n3000_d40": ("gauss", 3000, 40, 0), "movie_w7c1": ("movie", 7, 1, 1),
       "movie_w32c3": ("movie", 32, 3, 6)}
PCA_K = 6
NMF = {"n1500_d60_k5": (1500, 60, 5, 0), "n400_d100_k8": (400, 100, 8, 1),
       "n50_d200_k4": (50, 200, 4, 2)}                                   # (N, d, k, seed)
NMF_TOL = 1e-3     # the custom-init runs stop on the violation ratio well before max_iter
ICA = {"n2000_d8": (2000, 8, 0), "n3000_d5": (3000, 5, 1)}               # (N, d, seed), 3 sources
ICA_K = 3


def gauss(N, d, seed):
    """(N, d) float32 Gaussian cloud with a geometric, well-separated covariance spectrum."""
    rs = np.random.RandomState(seed)
    Q = np.linalg.qr(rs.randn(d, d))[0]
    scale = 3.0 * 0.8 ** np.arange(d)
    return (rs.randn(N, d) * scale @ Q.T + rs.randn(d)).astype(np.float32)


def movie_stack(window, channels, frames):
    """(n, window * window * channels) float32: the atom windows of stat_cases.separated_movie."""
    imgs, coords = stat_cases.separated_movie(window, channels, frames)
    out = []
    for f in range(frames):
        for x, y, c in coords[f]:
            if c != 0:
                continue
            x0, y0 = int(round(x)) - window // 2, int(round(y)) - window // 2
            out.append(imgs[f, x0:x0 + window, y0:y0 + window].ravel())
    return np.stack(out).astype(np.float32)


def pca_input(tag):
    kind, a, b, c = PCA[tag]
    return gauss(a, b, c) if kind == "gauss" else movie_stack(a, b, c)


def nmf_mixture(N, d, k, seed):
    """(N, d) float32 non-negative mixture of k smooth non-negative patterns, with noise, and a
    float32 starting point (W0, H0) drawn like sklearn's 'random' init."""
    rs = np.random.RandomState(seed)
    t = np.linspace(0, 1, d)
    H = np.stack([np.exp(-((t - c) / w) ** 2) for c, w in zip(rs.rand(k), 0.05 + 0.2 * rs.rand(k))])
    W = rs.exponential(1.0, (N, k))
    X = (W @ H + 0.02 * np.abs(rs.randn(N, d))).astype(np.float32)
    avg = np.sqrt(X.mean() / k)
    H0 = np.abs(avg * rs.randn(k, d)).astype(np.float32)
    W0 = np.abs(avg * rs.randn(N, k)).astype(np.float32)
    return X, W0, H0


def ica_mixture(N, d, seed):
    """(N, d) float32 mix of three non-Gaussian sources (Laplace, uniform, sine) plus small noise."""
    rs = np.random.RandomState(seed)
    t = np.linspace(0, 40, N)
    S = np.stack([rs.laplace(size=N), rs.uniform(-1, 1, N) * np.sqrt(3), np.sqrt(2) * np.sin(t)], 1)
    A = rs.randn(d, 3)
    return (S @ A.T + 0.01 * rs.randn(N, d) + rs.randn(d)).astype(np.float32)
