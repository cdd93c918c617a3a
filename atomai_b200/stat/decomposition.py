"""
Native PCA, NMF and FastICA over a stack of flattened sub-images or a hyperspectral matrix (the
subsets of sklearn.decomposition.PCA / NMF / FastICA that atomai.stat calls, with sklearn's
parameter names and defaults).

Every pass over the data runs in csrc/decomp.cu (and atomai_b200_stat_accum for W^T X and column
sums), in exact fp32 FFMA whatever set_math says, with float64 sums across rows:
  PCA      one Gram pass ((X - mean)^T (X - mean), or (X - mean)(X - mean)^T when N < d), then a
           float64 eigensolve of the Gram on the device;
  NMF      per coordinate-descent iteration one fused W sweep (X H^T and the W update) and one pass
           for W^T X, then the H sweep; one scalar is read back per iteration;
  FastICA  PCA whitening, one projection pass, then one pass over the whitened N x k samples per
           iteration; the k x k symmetric decorrelation runs in float64 on the host.
Inputs are (N, ...) numpy arrays or CUDA tensors (stacks are flattened); outputs are numpy arrays.
"""
import warnings

import numpy as np
import torch

from .. import _C, ops
from .mixture import MAX_COMPONENTS, _as_device, _check_k, _shape

_NMF_INITS = (None, "random", "nndsvd", "nndsvda", "custom")


def _rng(random_state):
    """sklearn's check_random_state"""
    if random_state is None:
        return np.random.mtrand._rand
    if isinstance(random_state, np.random.RandomState):
        return random_state
    return np.random.RandomState(random_state)


def _check_free(need: int, what: str) -> None:
    free, _ = torch.cuda.mem_get_info()
    if need > free:
        raise MemoryError(f"{what} needs about {need / 2**30:.1f} GiB of device memory, "
                          f"{free / 2**30:.1f} GiB are free; fit a subset of the data")


def _accum_bytes(N: int, d: int, k: int) -> int:
    """float64 ordered partials of atomai_b200_stat_accum (FFMA kernels: per 4096-row chunk and
    block of 32 columns, k x 65 values)"""
    return ((N + 4095) // 4096) * ((d + 31) // 32) * min(k, MAX_COMPONENTS) * 65 * 8


def _gram_bytes(N: int, d: int) -> int:
    """the m x m float64 Gram (m = min(N, d)) with room for the eigensolver's vectors and
    workspace, and the Gram pass's ordered partials"""
    m = min(N, d)
    return 4 * m * m * 8 + 8 * ops.decomp_slot_doubles(int(N < d), N, d, 1)


def _load(X, need: int, what: str) -> torch.Tensor:
    N, d = _shape(X)
    return _as_device(X, lambda copy: _check_free(need + (N * d * 4 if copy else 0), what))


def _sums(Xd: torch.Tensor, mu=None, squares: bool = False):
    """float64 column sums of X - mu (and of the squares)"""
    d = Xd.shape[1]
    sx = torch.empty(1, d, dtype=torch.float64, device=Xd.device)
    sxx = torch.empty_like(sx) if squares else None
    ops.stat_accum(Xd, mu, 1, sx, sxx, math=_C.MATH_FP32)
    return (sx[0], sxx[0]) if squares else sx[0]


def _weighted_rows(Xd: torch.Tensor, mu, R: torch.Tensor) -> torch.Tensor:
    """float64 (k, d) = R^T (X - mu) for R (N, k), k in blocks of MAX_COMPONENTS"""
    N, d = Xd.shape
    k = R.shape[1]
    out = torch.empty(k, d, dtype=torch.float64, device=Xd.device)
    for k0 in range(0, k, MAX_COMPONENTS):
        kb = min(MAX_COMPONENTS, k - k0)
        r = R[:, k0:k0 + kb].float().contiguous()
        ops.stat_accum(Xd, mu, kb, out[k0:k0 + kb], resp=r, math=_C.MATH_FP32)
    return out


def _project(Xd: torch.Tensor, mu, B) -> np.ndarray:
    out = torch.empty(Xd.shape[0], B.shape[0], device=Xd.device)
    ops.decomp_project(Xd, mu, B, out)
    return out.cpu().numpy()


def _top_eig(Xd: torch.Tensor, mu, k: int):
    """the k leading eigenpairs of the Gram of X - mu: eigenvalues (descending, clipped at 0) of
    all min(N, d), and the k unit feature-space vectors V (k, d) float64 on the device"""
    N, d = Xd.shape
    rows = N < d
    m = min(N, d)
    G = torch.empty(m, m, dtype=torch.float64, device=Xd.device)
    ops.decomp_gram(Xd, mu, G, rows)
    lam, vec = torch.linalg.eigh(G)
    del G
    lam, vec = lam.flip(0).clamp_min(0.0), vec.flip(1)[:, :k]
    if not rows:
        return lam, vec.T.contiguous()
    # N < d: the sample-space vectors U give V = (X - mu)^T U / s, normalised
    V = _weighted_rows(Xd, mu, vec)
    nrm = V.norm(dim=1, keepdim=True)
    return lam, torch.where(nrm > 0, V / nrm.clamp_min(1e-300), V)


def _bad_k(k, m: int, name: str = "n_components") -> int:
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)):
        raise NotImplementedError(f"{name}={k!r}: only an integer or None is supported")
    if not 1 <= k <= m:
        raise ValueError(f"{name}={k} must be between 1 and min(n_samples, n_features)={m}")
    return int(k)


class PCA:
    """Exact PCA (sklearn's full / covariance-eigh solvers) on the GPU.  `random_state` is
    accepted for signature compatibility and unused: the solver is exact."""

    def __init__(self, n_components=None, *, random_state=None):
        self.n_components = n_components
        self.random_state = random_state

    def _fit(self, X) -> torch.Tensor:
        N, d = _shape(X)
        if N < 2:
            raise ValueError(f"PCA needs at least 2 samples, got {N}")
        m = min(N, d)
        k = m if self.n_components is None else _bad_k(self.n_components, m)
        Xd = _load(X, _gram_bytes(N, d) + (N * k * 4 + k * d * 8 + _accum_bytes(N, d, k)
                                           if N < d else 0), f"PCA of {N} x {d}")
        mean = _sums(Xd) / N
        mu = mean.float().contiguous()
        lam, V = _top_eig(Xd, mu, k)
        # sklearn's svd_flip(u_based_decision=False): the largest |entry| of a component is > 0
        i = V.abs().argmax(1)
        V = V * torch.sign(V[torch.arange(k, device=V.device), i])[:, None]
        ev = lam / (N - 1)
        self.n_components_ = k
        self.n_samples_, self.n_features_in_ = N, d
        self.mean_ = mean.cpu().numpy()
        self.components_ = V.cpu().numpy()
        self.explained_variance_ = ev[:k].cpu().numpy()
        self.explained_variance_ratio_ = (ev[:k] / ev.sum()).cpu().numpy()
        self.singular_values_ = lam[:k].sqrt().cpu().numpy()
        self._mu, self._B = mu, V.float().contiguous()
        return Xd

    def fit(self, X, y=None):
        self._fit(X)
        return self

    def fit_transform(self, X, y=None) -> np.ndarray:
        return _project(self._fit(X), self._mu, self._B)

    def transform(self, X) -> np.ndarray:
        N, d = _shape(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, the model {self.n_features_in_}")
        Xd = _load(X, N * self.n_components_ * 4, f"PCA transform of {N} x {d}")
        return _project(Xd, self._mu, self._B)


def _nndsvd(U, S, V, avg, eps: float = 1e-6):
    """sklearn's NNDSVD from the top-k SVD U diag(S) V (float64 tensors); avg fills the zeros
    ('nndsvda') unless None ('nndsvd')"""
    W, H = torch.zeros_like(U), torch.zeros_like(V)
    W[:, 0] = S[0].sqrt() * U[:, 0].abs()
    H[0] = S[0].sqrt() * V[0].abs()
    for j in range(1, S.numel()):
        x, y = U[:, j], V[j]
        xp, yp, xn, yn = x.clamp_min(0), y.clamp_min(0), (-x).clamp_min(0), (-y).clamp_min(0)
        xpn, ypn, xnn, ynn = (float(a.norm()) for a in (xp, yp, xn, yn))
        mp, mn = xpn * ypn, xnn * ynn
        u, v, sigma = (xp / xpn, yp / ypn, mp) if mp > mn else (xn / xnn, yn / ynn, mn)
        lbd = (S[j] * sigma).sqrt()
        W[:, j], H[j] = lbd * u, lbd * v
    W[W < eps] = 0
    H[H < eps] = 0
    if avg is not None:
        W[W == 0] = avg
        H[H == 0] = avg
    return W, H


def _random_init(mean, N: int, d: int, k: int, random_state):
    """sklearn's 'random' NMF init for float32 X with X.mean() == mean: H then W from the same
    generator, scaled by sqrt(mean / k), absolute values"""
    avg = np.sqrt(np.float32(mean) / k)
    rng = _rng(random_state)
    H = np.abs(avg * rng.standard_normal(size=(k, d)).astype(np.float32))
    W = np.abs(avg * rng.standard_normal(size=(N, k)).astype(np.float32))
    return W, H


class NMF:
    """Non-negative matrix factorisation X ~ W H by coordinate descent (sklearn's 'cd' solver,
    Frobenius loss, no regularisation) on the GPU; k <= 64 components."""

    def __init__(self, n_components=None, *, init=None, max_iter=200, tol=1e-4, random_state=None):
        self.n_components = n_components
        self.init = init
        self.max_iter = max_iter
        self.tol = tol
        self.random_state = random_state

    def _k(self, d: int) -> int:
        return _check_k(d if self.n_components is None else self.n_components, "n_components")

    def _validate(self, X, W, H):
        N, d = _shape(X)
        k = self._k(d)
        if self.init == "nndsvdar":
            raise NotImplementedError("NMF: init='nndsvdar' is not native; use 'nndsvda'")
        if self.init not in _NMF_INITS:
            raise ValueError(f"invalid init {self.init!r}; use one of {_NMF_INITS}")
        if isinstance(self.max_iter, bool) or not isinstance(self.max_iter, (int, np.integer)) \
                or self.max_iter < 1 or self.tol < 0:
            raise ValueError("max_iter must be an integer >= 1 and tol >= 0")
        init = self.init
        if init is None:
            init = "nndsvda" if k <= min(N, d) else "random"
        if init in ("nndsvd", "nndsvda") and k > min(N, d):
            raise ValueError(f"init={init!r} needs n_components <= min(n_samples, n_features)")
        if init == "custom":
            if W is None or H is None or np.shape(W) != (N, k) or np.shape(H) != (k, d):
                raise ValueError(f"init='custom' needs W of shape {(N, k)} and H of shape {(k, d)}")
            for name, a in (("W", W), ("H", H)):
                if np.min(np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a)) < 0:
                    raise ValueError(f"Negative values in data passed to NMF (input {name})")
        if not (isinstance(X, torch.Tensor) and X.is_cuda) and np.min(np.asarray(X)) < 0:
            raise ValueError("Negative values in data passed to NMF (input X)")
        return N, d, k, init

    def _need(self, N: int, d: int, k: int, init: str) -> int:
        b = N * k * 4 + k * d * (4 + 8) + _accum_bytes(N, d, k)
        b += 8 * (ops.decomp_slot_doubles(2, N, d, k) + ops.decomp_slot_doubles(3, N, d, k))
        if init in ("nndsvd", "nndsvda"):
            b += _gram_bytes(N, d) + N * k * 8 * 3 + k * d * 8 * 3
        return b

    def _load(self, X, need: int) -> torch.Tensor:
        N, d = _shape(X)
        Xd = _load(X, need, f"NMF of {N} x {d}")
        if isinstance(X, torch.Tensor) and X.is_cuda and bool((Xd < 0).any()):
            raise ValueError("Negative values in data passed to NMF (input X)")
        return Xd

    def _initialise(self, Xd, init: str, k: int, W, H):
        N, d = Xd.shape
        dev = Xd.device
        if init == "custom":
            return (torch.as_tensor(np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a),
                                    dtype=torch.float32).to(dev).contiguous() for a in (W, H))
        mean = float(_sums(Xd).sum()) / (N * d)
        if init == "random":
            W0, H0 = _random_init(np.float32(mean), N, d, k, self.random_state)
            return torch.from_numpy(W0).to(dev), torch.from_numpy(H0).to(dev)
        # NNDSVD from the exact top-k SVD of the uncentred X
        lam, V = _top_eig(Xd, None, k)
        S = lam[:k].sqrt()
        U = torch.empty(N, k, device=dev)
        ops.decomp_project(Xd, None, V.float().contiguous(), U)
        U = U.double() / S.clamp_min(torch.finfo(torch.float64).tiny)
        W0, H0 = _nndsvd(U, S, V, mean if init == "nndsvda" else None)
        return W0.float().contiguous(), H0.float().contiguous()

    def _solve(self, Xd, W, H, update_h: bool):
        """sklearn's _fit_coordinate_descent; returns n_iter and (W^T X, W^T W, H H^T) of the
        final factors when H is updated"""
        N, d = Xd.shape
        k = H.shape[0]
        dev = Xd.device
        hh = torch.empty(k, k, dtype=torch.float64, device=dev)
        ops.decomp_gram(H, None, hh, rows=True)
        wout = torch.empty(k * k + 1, dtype=torch.float64, device=dev)
        hout = torch.empty_like(wout)
        WtX = torch.empty(k, d, dtype=torch.float64, device=dev) if update_h else None
        vinit = None
        for n_iter in range(1, self.max_iter + 1):
            ops.decomp_nmf_w(Xd, H, hh, W, wout)
            if update_h:
                ops.stat_accum(Xd, None, k, WtX, resp=W, math=_C.MATH_FP32)
                ops.decomp_nmf_h(WtX, wout[:k * k].view(k, k), H, hout)
                hh = hout[:k * k].view(k, k)
                v = float((wout[k * k] + hout[k * k]).item())
            else:
                v = float(wout[k * k].item())
            if n_iter == 1:
                vinit = v
            if vinit == 0 or v / vinit <= self.tol:
                break
        if n_iter == self.max_iter and self.tol > 0:
            warnings.warn(f"Maximum number of iterations {self.max_iter} reached. Increase it to "
                          "improve convergence.", RuntimeWarning)
        return n_iter, (WtX, wout[:k * k].view(k, k), hh)

    def fit_transform(self, X, y=None, W=None, H=None) -> np.ndarray:
        N, d, k, init = self._validate(X, W, H)
        Xd = self._load(X, self._need(N, d, k, init))
        W, H = self._initialise(Xd, init, k, W, H)
        n_iter, (WtX, WtW, HHt) = self._solve(Xd, W, H, True)
        # ||X - W H||_F from the final factors: ||X||^2 - 2 <W^T X, H> + <W^T W, H H^T>
        xx = _sums(Xd, squares=True)[1].sum()
        err2 = xx - 2 * (WtX * H.double()).sum() + (WtW * HHt).sum()
        self.reconstruction_err_ = float(err2.clamp_min(0).sqrt())
        self.n_iter_ = n_iter
        self.n_components_ = k
        self.n_features_in_ = d
        self.components_ = H.cpu().numpy()
        self._H = H
        return W.cpu().numpy()

    def fit(self, X, y=None, **params):
        self.fit_transform(X, **params)
        return self

    def transform(self, X) -> np.ndarray:
        """W for the fitted components: sklearn's W sweeps from W = 0 with H fixed"""
        N, d = _shape(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, the model {self.n_features_in_}")
        k = self.n_components_
        if not (isinstance(X, torch.Tensor) and X.is_cuda) and np.min(np.asarray(X)) < 0:
            raise ValueError("Negative values in data passed to NMF (input X)")
        Xd = self._load(X, N * k * 4 + 8 * ops.decomp_slot_doubles(2, N, d, k))
        W = torch.zeros(N, k, device=Xd.device)
        self._solve(Xd, W, self._H, False)
        return W.cpu().numpy()


def _sym_decorrelation(W):
    """(W W^T)^(-1/2) W in float64, as sklearn's _sym_decorrelation"""
    s, u = np.linalg.eigh(W @ W.T)
    s = np.clip(s, np.finfo(W.dtype).tiny, None)
    return np.linalg.multi_dot([u * (1.0 / np.sqrt(s)), u.T, W])


class FastICA:
    """FastICA (parallel, logcosh with alpha = 1, unit-variance whitening through PCA) on the GPU;
    k <= 64 components."""

    def __init__(self, n_components=None, *, algorithm="parallel", whiten="unit-variance",
                 fun="logcosh", max_iter=200, tol=1e-4, w_init=None, random_state=None):
        self.n_components = n_components
        self.algorithm = algorithm
        self.whiten = whiten
        self.fun = fun
        self.max_iter = max_iter
        self.tol = tol
        self.w_init = w_init
        self.random_state = random_state

    def _validate(self, X):
        for name, want in (("algorithm", "parallel"), ("whiten", "unit-variance"),
                           ("fun", "logcosh")):
            if getattr(self, name) != want:
                raise NotImplementedError(f"FastICA: {name}={getattr(self, name)!r}; only "
                                          f"{want!r} is native")
        N, d = _shape(X)
        if N < 2:
            raise ValueError(f"FastICA needs at least 2 samples, got {N}")
        m = min(N, d)
        k = m if self.n_components is None else self.n_components
        if isinstance(k, (int, np.integer)) and not isinstance(k, bool) and k > m:
            warnings.warn(f"n_components is too large: it will be set to {m}")
            k = m
        k = _check_k(k, "n_components")
        if isinstance(self.max_iter, bool) or not isinstance(self.max_iter, (int, np.integer)) \
                or self.max_iter < 1 or self.tol < 0:
            raise ValueError("max_iter must be an integer >= 1 and tol >= 0")
        if self.w_init is not None and np.shape(self.w_init) != (k, k):
            raise ValueError(f"w_init has invalid shape {np.shape(self.w_init)}, expected {(k, k)}")
        return N, d, k

    def _fit(self, X) -> torch.Tensor:
        N, d, k = self._validate(X)
        need = _gram_bytes(N, d) + N * k * 4 + 8 * ops.decomp_slot_doubles(4, N, d, k)
        if N < d:
            need += N * k * 4 + k * d * 8 + _accum_bytes(N, d, k)
        Xd = _load(X, need, f"FastICA of {N} x {d}")
        mean = _sums(Xd) / N
        mu = mean.float().contiguous()
        lam, V = _top_eig(Xd, mu, k)
        # sklearn: u (left singular vectors of (X - mean)^T) *= sign(u[0]); K = (u / s)^T[:k]
        V = V * torch.sign(V[:, :1])
        K = V / lam[:k].sqrt()[:, None]
        X1 = torch.empty(N, k, device=Xd.device)
        ops.decomp_project(Xd, mu, (K * np.sqrt(N)).float().contiguous(), X1)
        w_init = self.w_init
        if w_init is None:
            w_init = _rng(self.random_state).normal(size=(k, k))
        W = _sym_decorrelation(np.asarray(w_init, np.float64))
        out = torch.empty(k * k + k, dtype=torch.float64, device=Xd.device)
        for ii in range(self.max_iter):
            ops.decomp_ica_step(X1, torch.from_numpy(W).to(Xd.device), out)
            o = out.cpu().numpy()
            gx, gg = o[:k * k].reshape(k, k), o[k * k:]
            W1 = _sym_decorrelation(gx / N - (gg / N)[:, None] * W)
            lim = np.max(np.abs(np.abs(np.einsum("ij,ij->i", W1, W)) - 1))
            W = W1
            if lim < self.tol:
                break
        else:
            warnings.warn("FastICA did not converge. Consider increasing tolerance or the "
                          "maximum number of iterations.")
        # unit variance: the whitened samples have identity covariance, so the sources W K (x -
        # mean) have standard deviations sqrt(diag(W W^T) / N)
        s_std = np.sqrt(np.einsum("ij,ij->i", W, W) / N)
        W = W / s_std[:, None]
        K = K.cpu().numpy()
        self.n_iter_ = ii + 1
        self.components_ = W @ K
        self.mixing_ = np.linalg.pinv(self.components_)
        self.mean_ = mean.cpu().numpy()
        self.whitening_ = K
        self._unmixing = W
        self.n_features_in_ = d
        self._mu = mu
        self._B = torch.from_numpy(self.components_).float().to(Xd.device).contiguous()
        return Xd

    def fit(self, X, y=None):
        self._fit(X)
        return self

    def fit_transform(self, X, y=None) -> np.ndarray:
        return _project(self._fit(X), self._mu, self._B)

    def transform(self, X) -> np.ndarray:
        N, d = _shape(X)
        if d != self.n_features_in_:
            raise ValueError(f"X has {d} features, the model {self.n_features_in_}")
        Xd = _load(X, N * self._B.shape[0] * 4, f"FastICA transform of {N} x {d}")
        return _project(Xd, self._mu, self._B)
