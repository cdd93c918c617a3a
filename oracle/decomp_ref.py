"""
Float64 numpy restatement of the passes of csrc/decomp.cu and of the sklearn algorithms they serve
(PCA's Gram, NMF coordinate descent as sklearn's _update_cdnmf_fast / _fit_coordinate_descent,
NNDSVD(a) from a given SVD, FastICA's parallel logcosh step with its symmetric decorrelation): the
bound the GPU tests check the kernels against, and iterated here it reproduces sklearn's results.
"""
import numpy as np


def gram(X, mu=None, rows=False):
    """(X - mu)^T (X - mu), or (X - mu)(X - mu)^T when `rows`, in float64."""
    Xc = np.asarray(X, np.float64) - (0.0 if mu is None else np.asarray(mu, np.float64))
    return Xc @ Xc.T if rows else Xc.T @ Xc


def cd_update(W, HHt, XHt):
    """sklearn's _update_cdnmf_fast on W (n, k) in place: components in order, rows independent.
    Returns the summed projected-gradient violation."""
    violation = 0.0
    for t in range(W.shape[1]):
        grad = -XHt[:, t] + W @ HHt[t]
        pg = np.where(W[:, t] == 0, np.minimum(0.0, grad), grad)
        violation += np.abs(pg).sum()
        if HHt[t, t] != 0:
            W[:, t] = np.maximum(W[:, t] - grad / HHt[t, t], 0.0)
    return violation


def nmf_w_sweep(X, W, H):
    """one W sweep: the new W, its violation and W^T W of the new W."""
    X, W, H = (np.asarray(a, np.float64) for a in (X, W, H))
    W = W.copy()
    v = cd_update(W, H @ H.T, X @ H.T)
    return W, v, W.T @ W


def nmf_h_sweep(X, W, H):
    """one H sweep (W^T X and W^T W from the given W): the new H, its violation and H H^T."""
    X, W, H = (np.asarray(a, np.float64) for a in (X, W, H))
    Ht = H.T.copy()
    v = cd_update(Ht, W.T @ W, X.T @ W)
    return Ht.T, v, Ht.T @ Ht


def nmf_cd(X, W, H, tol=1e-4, max_iter=200, update_h=True):
    """sklearn's _fit_coordinate_descent (Frobenius, no regularisation): W, H, n_iter."""
    W, H = np.asarray(W, np.float64), np.asarray(H, np.float64)
    vinit = None
    for n_iter in range(1, max_iter + 1):
        W, v, _ = nmf_w_sweep(X, W, H)
        if update_h:
            H, vh, _ = nmf_h_sweep(X, W, H)
            v += vh
        if n_iter == 1:
            vinit = v
        if vinit == 0 or v / vinit <= tol:
            break
    return W, H, n_iter


def nndsvd(U, S, V, avg=None, eps=1e-6):
    """sklearn's NNDSVD from the top-k SVD X ~ U diag(S) V (U (n, k), V (k, d)); `avg` (X.mean())
    fills the zeros as 'nndsvda' does, None leaves them ('nndsvd')."""
    U, S, V = (np.asarray(a, np.float64) for a in (U, S, V))
    W, H = np.zeros_like(U), np.zeros_like(V)
    W[:, 0] = np.sqrt(S[0]) * np.abs(U[:, 0])
    H[0] = np.sqrt(S[0]) * np.abs(V[0])
    for j in range(1, len(S)):
        x, y = U[:, j], V[j]
        xp, yp, xn, yn = np.maximum(x, 0), np.maximum(y, 0), -np.minimum(x, 0), -np.minimum(y, 0)
        xpn, ypn, xnn, ynn = (np.linalg.norm(a) for a in (xp, yp, xn, yn))
        mp, mn = xpn * ypn, xnn * ynn
        u, v, sigma = (xp / xpn, yp / ypn, mp) if mp > mn else (xn / xnn, yn / ynn, mn)
        lbd = np.sqrt(S[j] * sigma)
        W[:, j], H[j] = lbd * u, lbd * v
    W[W < eps] = 0
    H[H < eps] = 0
    if avg is not None:
        W[W == 0] = avg
        H[H == 0] = avg
    return W, H


def sym_decorrelation(W):
    """(W W^T)^(-1/2) W, as sklearn's _sym_decorrelation."""
    s, u = np.linalg.eigh(W @ W.T)
    s = np.clip(s, np.finfo(W.dtype).tiny, None)
    return np.linalg.multi_dot([u * (1.0 / np.sqrt(s)), u.T, W])


def ica_sums(X1, W):
    """the kernel's sums over the whitened samples X1 (k, N): sum g x1^T and sum (1 - g^2), g =
    tanh(W x1)."""
    g = np.tanh(W @ X1)
    return g @ X1.T, (1.0 - g * g).sum(1)


def ica_step(X1, W):
    """one parallel logcosh FastICA step: W1 and lim = max | |diag(W1 W^T)| - 1 |."""
    gx, gg = ica_sums(X1, W)
    n = X1.shape[1]
    W1 = sym_decorrelation(gx / n - (gg / n)[:, None] * W)
    return W1, np.max(np.abs(np.abs(np.einsum("ij,ij->i", W1, W)) - 1))


def ica_par(X1, w_init, tol=1e-4, max_iter=200):
    """sklearn's _ica_par: W and the iteration count."""
    W = sym_decorrelation(np.asarray(w_init, np.float64))
    for ii in range(max_iter):
        W, lim = ica_step(X1, W)
        if lim < tol:
            break
    return W, ii + 1


def whitening(X, k):
    """FastICA's whitening (svd solver): mean, K (k x d) and X1 = K (X - mean)^T sqrt(N)."""
    X = np.asarray(X, np.float64)
    mean = X.mean(0)
    XT = (X - mean).T
    u, s = np.linalg.svd(XT, full_matrices=False)[:2]
    u *= np.sign(u[0])
    K = (u / s).T[:k]
    return mean, K, K @ XT * np.sqrt(X.shape[0])
