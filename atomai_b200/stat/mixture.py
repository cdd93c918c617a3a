"""
Native k-means and Gaussian-mixture estimators over a stack of flattened sub-images
(the subset of sklearn.cluster.KMeans / sklearn.mixture.GaussianMixture that
atomai.stat uses, atomai/stat/multivar.py:110-172, 816-900).

Every pass over the data runs in csrc/stat.cu: one E-step pass (responsibilities or
assignment) and one M-step pass (weighted sums) per iteration.  Each iteration reads one
scalar back for the convergence test; X and the responsibilities stay on the device.
Inputs are computed in fp32 (as sklearn computes the fp32 stacks Segmentor.predict returns).
"""
from typing import Optional, Union

import numpy as np
import torch

from .. import ops

MAX_COMPONENTS = 64          # K limit of the kernels (one warp lane pair per component)
_COVARIANCE_TYPES = ("diag", "spherical")


def _check_k(k, name: str) -> int:
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
        raise ValueError(f"{name} must be a positive integer, got {k!r}")
    if k > MAX_COMPONENTS:
        raise ValueError(f"{name} = {k} exceeds the native limit of {MAX_COMPONENTS} components")
    return int(k)


def _seed(random_state) -> int:
    if random_state is None:
        return int(np.random.randint(0, 2**31 - 1))
    if isinstance(random_state, np.random.RandomState):
        return int(random_state.randint(0, 2**31 - 1))
    return int(random_state)


def _shape(X):
    shape = tuple(X.shape)
    if len(shape) < 2:
        raise ValueError(f"expected a 2-D (n_samples, n_features) array or a stack, got shape {shape}")
    return shape[0], int(np.prod(shape[1:]))


def _check_memory(N: int, d: int, K: int, copy: bool) -> None:
    """Fails before anything is allocated when the fit's working set cannot fit in free memory:
    an fp32 copy of X (uploaded or converted), the N x K responsibilities, the N x (2 + ln K)
    k-means++ distances and other per-row buffers, and the M-step's float64 ordered partial sums
    (per 4096-row chunk and block of 32 columns: K x 65 values)."""
    ntr = 2 + int(np.log(K))
    partials = ((N + 4095) // 4096) * ((d + 31) // 32) * K * 65 * 8
    need = (N * d * 4 if copy else 0) + N * (K + ntr + 4) * 4 + partials + 4 * K * d * 8
    free, _ = torch.cuda.mem_get_info()
    if need > free:
        raise MemoryError(
            f"clustering {N} x {d} needs about {need / 2**30:.1f} GiB of device memory, "
            f"{free / 2**30:.1f} GiB are free; fit a subset of the stack")


def _device_matrix(X, K: int) -> torch.Tensor:
    N, d = _shape(X)
    if N < K:
        raise ValueError(f"n_samples={N} should be >= n_components={K}")
    return _as_device(X, lambda copy: _check_memory(N, d, K, copy))


def _as_device(X, check_memory) -> torch.Tensor:
    """X as a contiguous fp32 (N, d) CUDA tensor (X itself when it already is one), after
    check_memory(copy) has been told whether a copy of X is made."""
    N, d = _shape(X)
    if not torch.cuda.is_available():
        raise RuntimeError("atomai_b200.stat needs a CUDA device (there is no CPU path)")
    host = not (isinstance(X, torch.Tensor) and X.is_cuda)
    check_memory(host or X.dtype != torch.float32 or not X.is_contiguous())
    if host:
        X = torch.from_numpy(np.ascontiguousarray(np.asarray(X, dtype=np.float32)))
        return X.reshape(N, d).cuda()
    return X.detach().reshape(N, d).to(torch.float32).contiguous()


class _Centred:
    """X on the device with its column mean (float64 sums, fixed order) and mean column
    variance; the kernels subtract `mu` on every load."""

    def __init__(self, X: torch.Tensor):
        self.X = X
        self.N, self.d = X.shape
        dev = X.device
        sx = torch.empty(1, self.d, dtype=torch.float64, device=dev)
        sxx = torch.empty_like(sx)
        ops.stat_accum(X, None, 1, sx, sxx)
        mean = sx[0] / self.N
        self.mu = mean.float().contiguous()
        self.var_mean = float((sxx[0] / self.N - mean * mean).clamp_min(0).mean())


def _kmeans_plusplus(data: _Centred, K: int, seed: int) -> torch.Tensor:
    """Greedy k-means++ (sklearn's variant, 2 + int(ln K) candidates per step) with draws from the
    counter-hash generator; returns centred centres (K, d)."""
    X, mu, N, d = data.X, data.mu, data.N, data.d
    dev = X.device
    ntr = 2 + int(np.log(K))
    centres = torch.empty(K, d, device=dev)
    idx = torch.empty(ntr, dtype=torch.int32, device=dev)
    A = torch.empty(ntr, d, device=dev)
    cst = torch.empty(ntr, device=dev)
    pot = torch.empty(ntr, dtype=torch.float64, device=dev)
    closest = torch.empty(N, device=dev)
    labels = torch.zeros(N, dtype=torch.int32, device=dev)
    ops.stat_kpp_candidates(None, N, 1, seed, 0, None, idx)
    ops.stat_gather_rows(X, mu, idx[:1], centres[:1])
    ops.stat_kmeans_centres(centres[:1], A[:1], cst[:1])
    ops.stat_estep(X, mu, ops.STAT_KMEANS, A[:1], None, cst[:1], pot[:1], labels=labels,
                   rowval=closest)
    cand = torch.empty(ntr, d, device=dev)
    D = torch.empty(N, ntr, device=dev)
    ws = torch.empty(ops.stat_kpp_chunks(N), dtype=torch.float64, device=dev)
    for c in range(1, K):
        ops.stat_kpp_candidates(closest, N, ntr, seed, 32 * c, ws, idx)
        ops.stat_gather_rows(X, mu, idx, cand)
        ops.stat_kmeans_centres(cand, A, cst)
        ops.stat_estep(X, mu, ops.STAT_KPP, A, None, cst, pot, closest=closest, D=D)
        ops.stat_kpp_commit(D, pot, closest, cand, centres[c])
    return centres


def _lloyd(data: _Centred, centres: torch.Tensor, max_iter: int, tol: float):
    """sklearn's Lloyd loop on centred X: stop when no label changed or the squared centre shift
    is <= tol; the labels and inertia come from a last assignment with the final centres."""
    X, mu, N = data.X, data.mu, data.N
    K, d = centres.shape
    dev = X.device
    c, c_new = centres.contiguous(), torch.empty_like(centres)
    A = torch.empty(K, d, device=dev)
    cst = torch.empty(K, device=dev)
    sx = torch.empty(K, d, dtype=torch.float64, device=dev)
    nk = torch.empty(K, dtype=torch.float64, device=dev)
    status = torch.zeros(2, dtype=torch.float64, device=dev)     # label changes, centre shift
    out = torch.empty(1, dtype=torch.float64, device=dev)
    labels = torch.full((N,), -1, dtype=torch.int32, device=dev)
    ops.stat_kmeans_centres(c, A, cst)
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        status.zero_()
        ops.stat_estep(X, mu, ops.STAT_KMEANS, A, None, cst, out, labels=labels,
                       changes=status[:1])
        ops.stat_accum(X, mu, K, sx, nk=nk, labels=labels)
        ops.stat_kmeans_centres(c_new, A, cst, sx=sx, nk=nk, c_old=c, shift=status[1:])
        c, c_new = c_new, c
        changed, shift = status.tolist()
        if changed == 0 or shift <= tol:
            break
    ops.stat_estep(X, mu, ops.STAT_KMEANS, A, None, cst, out, labels=labels)
    return c, A, cst, labels, float(out.item()), n_iter


class KMeans:
    """k-means (Lloyd) with greedy k-means++ seeding on the GPU; the sklearn.cluster.KMeans
    subset atomai uses.  One initialisation (n_init must be 1 or 'auto')."""

    def __init__(self, n_clusters: int = 8, *, init: Union[str, np.ndarray] = "k-means++",
                 n_init: Union[str, int] = "auto", max_iter: int = 300, tol: float = 1e-4,
                 random_state=None):
        self.n_clusters = n_clusters
        self.init = init
        self.n_init = n_init
        self.max_iter = max_iter
        self.tol = tol
        self.random_state = random_state

    def _validate(self, X):
        K = _check_k(self.n_clusters, "n_clusters")
        if self.n_init not in ("auto", 1):
            raise NotImplementedError("KMeans: only one initialisation (n_init=1 or 'auto') is native")
        if isinstance(self.init, str):
            if self.init != "k-means++":
                raise NotImplementedError(f"KMeans: init={self.init!r}; use 'k-means++' or an array")
        elif np.shape(self.init) != (K, _shape(X)[1]):
            raise ValueError(f"init array must have shape {(K, _shape(X)[1])}, got {np.shape(self.init)}")
        if self.max_iter < 1:
            raise ValueError(f"max_iter must be >= 1, got {self.max_iter}")
        return K

    def fit(self, X, y=None):
        K = self._validate(X)
        data = _Centred(_device_matrix(X, K))
        if isinstance(self.init, str):
            centres = _kmeans_plusplus(data, K, _seed(self.random_state))
        else:
            init = torch.as_tensor(np.asarray(self.init, dtype=np.float32), device=data.X.device)
            centres = (init - data.mu).contiguous()
        c, self._A, self._cst, labels, self.inertia_, self.n_iter_ = _lloyd(
            data, centres, self.max_iter, self.tol * data.var_mean)
        self._mu = data.mu
        self._labels = labels
        self.cluster_centers_ = (c + data.mu).cpu().numpy()
        self.labels_ = labels.cpu().numpy().astype(np.int64)
        return self

    def fit_predict(self, X, y=None) -> np.ndarray:
        return self.fit(X).labels_

    def predict(self, X) -> np.ndarray:
        Xd = _device_matrix(X, 1)
        if Xd.shape[1] != self._A.shape[1]:
            raise ValueError(f"X has {Xd.shape[1]} features, the model {self._A.shape[1]}")
        labels = torch.full((Xd.shape[0],), -1, dtype=torch.int32, device=Xd.device)
        out = torch.empty(1, dtype=torch.float64, device=Xd.device)
        ops.stat_estep(Xd, self._mu, ops.STAT_KMEANS, self._A, None, self._cst, out, labels=labels)
        return labels.cpu().numpy().astype(np.int64)


class GaussianMixture:
    """EM for a Gaussian mixture with 'diag' or 'spherical' covariances on the GPU, initialised
    like sklearn (hard labels of one k-means run) or from `init_labels` (an N-vector of initial
    hard assignments, which replaces the k-means seeding)."""

    def __init__(self, n_components: int = 1, *, covariance_type: str = "full", tol: float = 1e-3,
                 reg_covar: float = 1e-6, max_iter: int = 100, init_params: str = "kmeans",
                 random_state=None, init_labels: Optional[np.ndarray] = None):
        self.n_components = n_components
        self.covariance_type = covariance_type
        self.tol = tol
        self.reg_covar = reg_covar
        self.max_iter = max_iter
        self.init_params = init_params
        self.random_state = random_state
        self.init_labels = init_labels

    def _validate(self, X):
        K = _check_k(self.n_components, "n_components")
        if self.covariance_type in ("full", "tied"):
            raise NotImplementedError(
                f"covariance_type={self.covariance_type!r} is not on the native path; "
                "use 'diag' or 'spherical'")
        if self.covariance_type not in _COVARIANCE_TYPES:
            raise ValueError(f"invalid covariance_type {self.covariance_type!r}")
        if self.init_params != "kmeans":
            raise NotImplementedError(f"init_params={self.init_params!r}; only 'kmeans' is native")
        if self.max_iter < 1 or self.reg_covar < 0 or self.tol < 0:
            raise ValueError("max_iter must be >= 1 and reg_covar, tol >= 0")
        if self.init_labels is not None:
            lab = np.asarray(self.init_labels)
            if lab.shape != (_shape(X)[0],) or lab.min() < 0 or lab.max() >= K:
                raise ValueError(f"init_labels must be {_shape(X)[0]} integers in [0, {K})")
        return K

    def fit(self, X, y=None):
        self.fit_predict(X)
        return self

    def fit_predict(self, X, y=None) -> np.ndarray:
        K = self._validate(X)
        data = _Centred(_device_matrix(X, K))
        Xd, mu, N, d = data.X, data.mu, data.N, data.d
        dev = Xd.device
        if self.init_labels is not None:
            labels = torch.as_tensor(np.asarray(self.init_labels, dtype=np.int32), device=dev)
        else:
            km = KMeans(K, n_init=1, random_state=self.random_state)
            labels = _lloyd(data, _kmeans_plusplus(data, K, _seed(self.random_state)),
                            km.max_iter, km.tol * data.var_mean)[3]
        sph = self.covariance_type == "spherical"
        sx = torch.empty(K, d, dtype=torch.float64, device=dev)
        sxx = torch.empty_like(sx)
        nk = torch.empty(K, dtype=torch.float64, device=dev)
        means = torch.empty(K, d, device=dev)
        covs = torch.empty(K if sph else (K, d), device=dev)
        weights = torch.empty(K, device=dev)
        A, B = torch.empty(K, d, device=dev), torch.empty(K, d, device=dev)
        cst = torch.empty(K, device=dev)
        resp = torch.empty(N, K, device=dev)
        out = torch.empty(1, dtype=torch.float64, device=dev)
        params = (means, covs, weights, A, B, cst)
        ops.stat_accum(Xd, mu, K, sx, sxx, nk, labels=labels)
        ops.stat_gmm_params(sx, sxx, nk, N, sph, self.reg_covar, 1, *params)
        lb, self.lower_bounds_, self.converged_ = -np.inf, [], False
        for n_iter in range(1, self.max_iter + 1):
            prev = lb
            ops.stat_estep(Xd, mu, ops.STAT_GMM, A, B, cst, out, resp=resp)
            ops.stat_accum(Xd, mu, K, sx, sxx, nk, resp=resp)
            ops.stat_gmm_params(sx, sxx, nk, N, sph, self.reg_covar, 0, *params)
            lb = out.item() / N
            self.lower_bounds_.append(lb)
            if abs(lb - prev) < self.tol:
                self.converged_ = True
                break
        self.n_iter_, self.lower_bound_ = n_iter, lb
        self._mu, self._A, self._B, self._cst = mu, A, B, cst
        self.means_ = (means + mu).cpu().numpy()
        self.covariances_ = covs.cpu().numpy()
        self.weights_ = weights.cpu().numpy()
        self.precisions_cholesky_ = 1.0 / np.sqrt(self.covariances_)
        return self._predict_device(Xd)

    def _predict_device(self, Xd: torch.Tensor) -> np.ndarray:
        labels = torch.empty(Xd.shape[0], dtype=torch.int32, device=Xd.device)
        out = torch.empty(1, dtype=torch.float64, device=Xd.device)
        ops.stat_estep(Xd, self._mu, ops.STAT_GMM, self._A, self._B, self._cst, out, labels=labels)
        return labels.cpu().numpy().astype(np.int64)

    def predict(self, X) -> np.ndarray:
        Xd = _device_matrix(X, 1)
        if Xd.shape[1] != self._A.shape[1]:
            raise ValueError(f"X has {Xd.shape[1]} features, the model {self._A.shape[1]}")
        return self._predict_device(Xd)
