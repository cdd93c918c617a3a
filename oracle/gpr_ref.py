"""
TEST INFRASTRUCTURE — float64 numpy / scipy restatement of the Reconstructor's exact GP
(atomai/models/dklgp/gpr.py, atomai/trainers/gptrainer.py:59-137, atomai/nets/gp.py:63-128 with the
kernel formulas of oracle/gram_ref.py and gpytorch's parametrisation as atomai_b200.nets.gp.
CustomGPModel restates it):
  lengthscale = softplus(raw) | lower + (upper - lower) sigmoid(raw),  outputscale = softplus(raw),
  noise = softplus(raw) + 1e-4,  mean = raw constant;
  loss = -log N(y; c, K + noise I) / N;  Adam as torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8).
Distances are formed from coordinate differences, never from a norm expansion.  gpytorch is not
installed here, so parity with it is UNPINNED; the gradients are pinned to finite differences.
"""
import numpy as np
from scipy.linalg import cho_factor, cho_solve

RAW_KEYS = ("ls", "os", "noise", "c")


def softplus(x):
    return np.logaddexp(0.0, x)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def hyper(raw, bounds=None):
    """Constrained hyper-parameters from the raw dict {ls: (d,), os, noise, c}."""
    ls_raw = np.asarray(raw["ls"], np.float64)
    if bounds is None:
        ls = softplus(ls_raw)
    else:
        lo, hi = (np.asarray(b, np.float64) for b in bounds)
        ls = lo + (hi - lo) * sigmoid(ls_raw)
    return dict(ls=ls, os=float(softplus(raw["os"])), noise=float(softplus(raw["noise"]) + 1e-4),
                c=float(raw["c"]))


def _r2(x1, x2, ls):
    diff = (np.asarray(x1, np.float64)[:, None, :] - np.asarray(x2, np.float64)[None, :, :]) / ls
    return diff, (diff * diff).sum(-1)


def kernel(x1, x2, ls, os, kind="rbf"):
    _, r2 = _r2(x1, x2, ls)
    if kind == "rbf":
        return os * np.exp(-0.5 * r2)
    s = np.sqrt(5.0 * r2)
    return os * (1.0 + s + 5.0 / 3.0 * r2) * np.exp(-s)


def kernel_grads(x1, x2, ls, os, kind="rbf"):
    """K and its derivatives: dK/dls (d, n1, n2), dK/dos (n1, n2), dK/dx1 (n1, n2, d)."""
    diff, r2 = _r2(x1, x2, ls)
    if kind == "rbf":
        K = os * np.exp(-0.5 * r2)
        m = K                                   # -2 dK/dr^2
    else:
        s = np.sqrt(5.0 * r2)
        K = os * (1.0 + s + 5.0 / 3.0 * r2) * np.exp(-s)
        m = 5.0 / 3.0 * os * (1.0 + s) * np.exp(-s)
    dls = m[None] * np.moveaxis(diff * diff, -1, 0) / np.asarray(ls)[:, None, None]
    dx1 = -m[..., None] * diff / np.asarray(ls)
    return K, dls, K / os, dx1


def neg_mll(x, y, p, kind="rbf"):
    n = len(y)
    Kn = kernel(x, x, p["ls"], p["os"], kind) + p["noise"] * np.eye(n)
    cf = cho_factor(Kn, lower=True)
    r = np.asarray(y, np.float64) - p["c"]
    alpha = cho_solve(cf, r)
    logdet = 2.0 * np.log(np.diag(cf[0])).sum()
    return (0.5 * r @ alpha + 0.5 * logdet + 0.5 * n * np.log(2 * np.pi)) / n


def neg_mll_grad(x, y, p, kind="rbf"):
    """Gradient of neg_mll w.r.t. the constrained hyper-parameters:
    d/dtheta = tr((Kn^-1 - alpha alpha^T) dKn/dtheta) / (2N),  d/dc = -sum(alpha) / N."""
    n = len(y)
    K, dls, dos, _ = kernel_grads(x, x, p["ls"], p["os"], kind)
    Kn = K + p["noise"] * np.eye(n)
    cf = cho_factor(Kn, lower=True)
    alpha = cho_solve(cf, np.asarray(y, np.float64) - p["c"])
    A = cho_solve(cf, np.eye(n)) - np.outer(alpha, alpha)
    return dict(ls=np.array([(A * g).sum() for g in dls]) / (2 * n),
                os=float((A * dos).sum()) / (2 * n), noise=float(np.trace(A)) / (2 * n),
                c=float(-alpha.sum()) / n)


def raw_grad(x, y, raw, kind="rbf", bounds=None):
    """Gradient of neg_mll w.r.t. the raw parameters (chain rule through the transforms)."""
    p = hyper(raw, bounds)
    g = neg_mll_grad(x, y, p, kind)
    ls_raw = np.asarray(raw["ls"], np.float64)
    if bounds is None:
        dls = sigmoid(ls_raw)
    else:
        lo, hi = (np.asarray(b, np.float64) for b in bounds)
        dls = (hi - lo) * sigmoid(ls_raw) * (1.0 - sigmoid(ls_raw))
    return dict(ls=g["ls"] * dls, os=g["os"] * sigmoid(raw["os"]),
                noise=g["noise"] * sigmoid(raw["noise"]), c=g["c"])


def posterior_mean(x, y, p, xq, kind="rbf"):
    n = len(y)
    Kn = kernel(x, x, p["ls"], p["os"], kind) + p["noise"] * np.eye(n)
    alpha = cho_solve(cho_factor(Kn, lower=True), np.asarray(y, np.float64) - p["c"])
    return p["c"] + kernel(xq, x, p["ls"], p["os"], kind) @ alpha


def initial_raw(d):
    return dict(ls=np.zeros(d), os=0.0, noise=0.0, c=0.0)


def fit(x, y, steps, lr=0.1, kind="rbf", bounds=None, raw=None):
    """`steps` Adam steps (torch.optim.Adam's update) on every raw parameter from `raw` (default:
    gpytorch's zeros); returns the final raw dict and the loss before each step."""
    raw = {k: np.array(v, np.float64) for k, v in (raw or initial_raw(x.shape[1])).items()}
    m = {k: np.zeros_like(v) for k, v in raw.items()}
    v = {k: np.zeros_like(v) for k, v in raw.items()}
    b1, b2, eps = 0.9, 0.999, 1e-8
    losses = []
    for t in range(1, steps + 1):
        losses.append(neg_mll(x, y, hyper(raw, bounds), kind))
        g = raw_grad(x, y, raw, kind, bounds)
        for k in RAW_KEYS:
            m[k] = b1 * m[k] + (1 - b1) * g[k]
            v[k] = b2 * v[k] + (1 - b2) * g[k] ** 2
            denom = np.sqrt(v[k]) / np.sqrt(1 - b2 ** t) + eps
            raw[k] = raw[k] - lr / (1 - b1 ** t) * m[k] / denom
    return raw, losses


def reconstruct(sparse_image, steps, lr=0.1, kind="rbf"):
    """Reconstructor.reconstruct in float64: fit on the non-zero pixels with the lengthscale
    bounded to [1, max index // 2 + 1], then the mean at every pixel (row-major)."""
    img = np.asarray(sparse_image)
    x = np.argwhere(img != 0).astype(np.float64)
    y = img[img != 0].astype(np.float64)
    full = np.indices(img.shape).reshape(img.ndim, -1).T.astype(np.float64)
    bounds = (np.ones(img.ndim), full.max(0) // 2 + 1)
    raw, _ = fit(x, y, steps, lr, kind, bounds)
    return posterior_mean(x, y, hyper(raw, bounds), full, kind).reshape(img.shape)
