"""
Float64 numpy restatement of one Lloyd step and one diagonal / spherical EM step (sklearn's
KMeans / GaussianMixture algebra), the bound for the kernels of csrc/stat.cu.  X is centred by the
caller the way the kernels centre it (by its column mean).
"""
import numpy as np

EPS10 = 10 * np.finfo(np.float32).eps


def sqdist(X, C):
    """(N, K) squared distances, float64, by the expansion (accurate in float64)."""
    X, C = np.asarray(X, np.float64), np.asarray(C, np.float64)
    return np.maximum((X * X).sum(1)[:, None] - 2 * X @ C.T + (C * C).sum(1)[None], 0.0)


def lloyd_step(X, C):
    """labels (first argmin), min distance, per-cluster sums and counts, inertia."""
    d2 = sqdist(X, C)
    lab = d2.argmin(1)
    K = len(C)
    onehot = np.eye(K)[lab]
    return lab, d2[np.arange(len(X)), lab], onehot.T @ np.asarray(X, np.float64), onehot.sum(0), \
        d2[np.arange(len(X)), lab].sum()


def log_gauss(X, means, covs, weights):
    """(N, K) weighted log densities; covs (K, d) diagonal or (K,) spherical."""
    X = np.asarray(X, np.float64)
    means = np.asarray(means, np.float64)
    covs = np.asarray(covs, np.float64)
    if covs.ndim == 1:
        covs = np.repeat(covs[:, None], X.shape[1], 1)
    lp = np.stack([-0.5 * (((X - m) ** 2) / v + np.log(2 * np.pi * v)).sum(1)
                   for m, v in zip(means, covs)], 1)
    return lp + np.log(np.asarray(weights, np.float64))[None]


def e_step(X, means, covs, weights):
    """responsibilities, log_prob_norm per row."""
    lw = log_gauss(X, means, covs, weights)
    m = lw.max(1, keepdims=True)
    lse = (m + np.log(np.exp(lw - m).sum(1, keepdims=True)))[:, 0]
    return np.exp(lw - lse[:, None]), lse


def m_step(X, resp, reg_covar, covariance_type, init=False):
    """sklearn's _estimate_gaussian_parameters + weights (/ N at init, else normalised)."""
    X = np.asarray(X, np.float64)
    resp = np.asarray(resp, np.float64)
    nk = resp.sum(0) + EPS10
    means = resp.T @ X / nk[:, None]
    covs = resp.T @ (X * X) / nk[:, None] - 2 * means * (resp.T @ X) / nk[:, None] + means ** 2 \
        + reg_covar
    if covariance_type == "spherical":
        covs = covs.mean(1)
    weights = nk / (len(X) if init else nk.sum())
    return means, covs, weights
