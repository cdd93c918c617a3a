"""atomai_b200.stat PCA / NMF / FastICA on the GPU: each pass of csrc/decomp.cu against the float64
restatement (oracle/decomp_ref.py) within bounds derived from the fp32 rounding of its sums,
bit-reproducibility, and the estimators against sklearn (tests/golden/decomp_sklearn.npz)."""
import os

import numpy as np
import pytest
import torch

import decomp_cases as dc
from atomai_b200 import ops, stat
from oracle import decomp_ref

pytestmark = pytest.mark.gpu
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SK = np.load(os.path.join(HERE, "decomp_sklearn.npz"))
EPS32 = float(np.finfo(np.float32).eps)


def _dot_tol(L, mag):
    """bound on an fp32 L-term sum whose terms have magnitudes summing to `mag` (as in
    test_stat_gpu.py): 8 sqrt(L) eps per unit of magnitude"""
    return 8 * np.sqrt(L) * EPS32 * mag


def _data(N, d, seed, nonneg=False):
    rs = np.random.RandomState(seed)
    X = rs.randn(N, d) * (0.5 + rs.rand(d)) + 3.0
    return (np.abs(X) if nonneg else X).astype(np.float32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


GRAM_CASES = [(1, 50), (63, 50), (63, 200), (4097, 70), (4097, 130), (2 ** 17 + 3, 49), (300, 3072)]


@pytest.mark.parametrize("N,d", GRAM_CASES)
@pytest.mark.parametrize("rows", [False, True])
def test_gram_matches_float64(cuda, N, d, rows):
    if rows and N > 4097:
        pytest.skip("N x N Gram too large for the float64 reference")
    X = _data(N, d, 0)
    mu = X.mean(0).astype(np.float32)
    m = N if rows else d
    G = torch.empty(m, m, dtype=torch.float64, device=cuda)
    ops.decomp_gram(_dev(X), _dev(mu), G, rows)
    got = G.cpu().numpy()
    Xc = X.astype(np.float64) - mu
    ref = decomp_ref.gram(X, mu, rows)
    A = np.abs(Xc)
    mag = A @ A.T if rows else A.T @ A
    np.testing.assert_array_equal(got, got.T)
    assert np.all(np.abs(got - ref) <= _dot_tol(d if rows else N, mag) + 1e-30)
    G2 = torch.empty_like(G)
    ops.decomp_gram(_dev(X), _dev(mu), G2, rows)
    assert torch.equal(G, G2)


@pytest.mark.parametrize("N,d,k", [(1, 50, 1), (63, 49, 64), (4097, 70, 5), (2 ** 17 + 3, 49, 17),
                                   (300, 3072, 64), (100, 33, 70)])
def test_project_matches_float64(cuda, N, d, k):
    X = _data(N, d, 1)
    B = np.random.RandomState(2).randn(k, d).astype(np.float32)
    mu = X.mean(0).astype(np.float32)
    out = torch.empty(N, k, device=cuda)
    ops.decomp_project(_dev(X), _dev(mu), _dev(B), out)
    Xc = X.astype(np.float64) - mu
    ref = Xc @ B.T.astype(np.float64)
    assert np.all(np.abs(out.cpu().numpy() - ref) <= _dot_tol(d, np.abs(Xc) @ np.abs(B.T)) + 1e-30)


def _cd_bound(W, HHt, tau):
    """per-entry bound on a coordinate-descent sweep whose XHt entries are off by up to tau and
    whose updates are rounded to fp32: delta_t = (tau_t + sum_r HHt_tr delta_r) / HHt_tt + eps |w_t|"""
    delta = np.zeros_like(W)
    for t in range(W.shape[1]):
        h = HHt[t, t]
        delta[:, t] = (tau[:, t] + delta @ np.abs(HHt[t])) / h + 2 * EPS32 * np.abs(W[:, t]) \
            if h != 0 else 0.0
    return delta


SWEEP_CASES = [(1, 50, 1), (63, 49, 64), (4097, 70, 5), (4097, 33, 64), (2 ** 17 + 3, 49, 17)]


@pytest.mark.parametrize("N,d,k", SWEEP_CASES)
def test_nmf_w_sweep_matches_float64(cuda, N, d, k):
    X = _data(N, d, 3, nonneg=True)
    rs = np.random.RandomState(4)
    W0 = rs.rand(N, k).astype(np.float32)
    H = rs.rand(k, d).astype(np.float32)
    W0[rs.rand(N, k) < 0.2] = 0                   # exercise the projected gradient at W = 0
    HHt = H.astype(np.float64) @ H.T
    W = _dev(W0)
    out = torch.empty(k * k + 1, dtype=torch.float64, device=cuda)
    ops.decomp_nmf_w(_dev(X), _dev(H), _dev(HHt), W, out)
    Wr, vr, _ = decomp_ref.nmf_w_sweep(X, W0, H)
    tau = _dot_tol(d, X.astype(np.float64) @ H.T)
    delta = _cd_bound(Wr, HHt, tau)
    got = W.cpu().numpy()
    assert np.all(np.abs(got - Wr) <= 2 * delta + 1e-30)
    o = out.cpu().numpy()
    g64 = got.astype(np.float64)
    np.testing.assert_allclose(o[:k * k].reshape(k, k), g64.T @ g64, rtol=1e-12, atol=1e-300)
    gerr = (tau + delta @ np.abs(HHt)).sum()         # bound on the summed |grad| error
    assert abs(o[-1] - vr) <= 2 * gerr + 1e-9 * vr


@pytest.mark.parametrize("N,d,k", SWEEP_CASES)
def test_nmf_h_sweep_matches_float64(cuda, N, d, k):
    X = _data(N, d, 5, nonneg=True)
    rs = np.random.RandomState(6)
    W = rs.rand(N, k).astype(np.float32)
    H0 = rs.rand(k, d).astype(np.float32)
    W64 = W.astype(np.float64)
    WtX, WtW = W64.T @ X, W64.T @ W64
    H = _dev(H0)
    out = torch.empty(k * k + 1, dtype=torch.float64, device=cuda)
    ops.decomp_nmf_h(_dev(WtX), _dev(WtW), H, out)
    Hr, vr, _ = decomp_ref.nmf_h_sweep(X, W, H0)
    delta = _cd_bound(Hr.T, WtW, np.zeros((d, k))).T
    got = H.cpu().numpy()
    assert np.all(np.abs(got - Hr) <= 2 * delta + 1e-30)
    o = out.cpu().numpy()
    g64 = got.astype(np.float64)
    np.testing.assert_allclose(o[:k * k].reshape(k, k), g64 @ g64.T, rtol=1e-12, atol=1e-300)
    assert abs(o[-1] - vr) <= 2 * (delta.T @ np.abs(WtW)).sum() + 1e-9 * vr


@pytest.mark.parametrize("N,k", [(1, 1), (63, 64), (4097, 5), (4097, 64), (2 ** 17 + 3, 17)])
def test_ica_step_matches_float64(cuda, N, k):
    rs = np.random.RandomState(7)
    X1 = rs.laplace(size=(N, k)).astype(np.float32)
    W = decomp_ref.sym_decorrelation(rs.randn(k, k))
    out = torch.empty(k * k + k, dtype=torch.float64, device=cuda)
    ops.decomp_ica_step(_dev(X1), _dev(W), out)
    gx, gg = decomp_ref.ica_sums(X1.T.astype(np.float64), W)
    o = out.cpu().numpy()
    mag = np.abs(np.tanh(W @ X1.T)) @ np.abs(X1)
    np.testing.assert_allclose(o[:k * k].reshape(k, k), gx, rtol=0, atol=1e-12 * mag.max() + 1e-300)
    np.testing.assert_allclose(o[k * k:], gg, rtol=1e-12)


def _pca_bounds(X):
    """||tau||_F of the fp32 Gram pass (bounds every eigenvalue's error) for the float64 X"""
    N, d = X.shape
    A = np.abs(X - X.mean(0))
    mag = A @ A.T if N < d else A.T @ A
    return np.linalg.norm(_dot_tol(d if N < d else N, mag))


@pytest.mark.parametrize("tag", list(dc.PCA))
def test_pca_matches_sklearn(cuda, tag):
    X = dc.pca_input(tag)
    N, d = X.shape
    p = stat.PCA(random_state=0).fit(X)
    pre = f"pca/{tag}/"
    ev = SK[pre + "explained_variance"]
    tg = _pca_bounds(X.astype(np.float64))
    assert p.n_components_ == min(N, d) == len(ev)
    np.testing.assert_allclose(p.explained_variance_, ev, rtol=0, atol=2 * tg / (N - 1) + 1e-12 * ev[0])
    np.testing.assert_allclose(p.singular_values_ ** 2, SK[pre + "singular_values"] ** 2, rtol=0,
                               atol=2 * tg + 1e-12 * ev[0] * N)
    np.testing.assert_allclose(p.explained_variance_ratio_, SK[pre + "explained_variance_ratio"],
                               rtol=0, atol=4 * tg / (N - 1) / ev.sum())
    np.testing.assert_allclose(p.mean_, SK[pre + "mean"], rtol=0, atol=1e-6 * np.abs(X).max())
    lam = ev * (N - 1)
    q = stat.PCA(dc.PCA_K).fit(X)
    Z = q.transform(X)
    np.testing.assert_array_equal(Z, stat.PCA(dc.PCA_K).fit_transform(X))
    Xc = X.astype(np.float64) - SK[pre + "mean"]
    for i in range(dc.PCA_K):
        gap = min(abs(lam[i] - lam[j]) for j in range(len(lam)) if j != i)
        if gap < 1e3 * tg:
            continue                                   # not well separated at fp32 scale
        # sin(angle) <= ||dG|| / gap, plus the fp32 sums forming the vector when N < d
        tv = 4 * tg / gap + (2e-5 if N < d else 0.0)
        np.testing.assert_allclose(q.components_[i], SK[pre + "components"][i], rtol=0, atol=tv)
        tz = np.abs(Xc) @ np.full(d, tv) + _dot_tol(d, np.abs(Xc) @ np.abs(q.components_[i]))
        assert np.all(np.abs(Z[:, i] - SK[pre + "transform"][:, i]) <= tz)


def test_pca_cuda_input_and_repeat_bits(cuda):
    X = dc.pca_input("gauss_n3000_d40")
    a = stat.PCA(5).fit(X)
    b = stat.PCA(5).fit(torch.from_numpy(X).cuda().reshape(3000, 5, 8))
    for att in ("components_", "explained_variance_", "singular_values_", "mean_"):
        assert np.array_equal(getattr(a, att), getattr(b, att)), att


def _oracle_ratios(X, W0, H0, n):
    """violation / violation_init of the float64 trajectory for n iterations"""
    W, H = W0.astype(np.float64), H0.astype(np.float64)
    out = []
    for _ in range(n):
        W, vw, _ = decomp_ref.nmf_w_sweep(X, W, H)
        H, vh, _ = decomp_ref.nmf_h_sweep(X, W, H)
        out.append(vw + vh)
    return np.array(out) / out[0]


@pytest.mark.parametrize("tag", list(dc.NMF))
def test_nmf_follows_sklearn_from_custom_init(cuda, tag):
    N, d, k, seed = dc.NMF[tag]
    X, W0, H0 = dc.nmf_mixture(N, d, k, seed)
    m = stat.NMF(k, init="custom", tol=dc.NMF_TOL)
    W = m.fit_transform(X, W=W0, H=H0)
    pre = f"nmf/{tag}/"
    n_ref = int(SK[pre + "n_iter"])
    if m.n_iter_ != n_ref:
        r = _oracle_ratios(X, W0, H0, max(m.n_iter_, n_ref))
        lo = min(m.n_iter_, n_ref)
        assert np.all(np.abs(r[lo - 1:] / dc.NMF_TOL - 1) <= 0.02), (m.n_iter_, n_ref)
    Wr, Hr = SK[pre + "W"], SK[pre + "H"]
    assert np.abs(W - Wr).max() <= 2e-3 * np.abs(Wr).max()
    assert np.abs(m.components_ - Hr).max() <= 2e-3 * np.abs(Hr).max()
    np.testing.assert_allclose(m.reconstruction_err_, SK[pre + "err"], rtol=1e-3)
    # the expansion ||X||^2 - 2 <W^T X, H> + <W^T W, H H^T> of the fitted factors: its fp32 row
    # sums (chunks of up to 4096 rows) are off by a share of ||X||^2, not of the residual
    direct = np.linalg.norm(X - W.astype(np.float64) @ m.components_)
    xx = (X.astype(np.float64) ** 2).sum()
    assert abs(m.reconstruction_err_ ** 2 - direct ** 2) <= _dot_tol(min(N, 4096), xx)
    # transform: W sweeps from W = 0 against the fitted H, as the float64 restatement runs them
    Wt = m.transform(X)
    Wtr = decomp_ref.nmf_cd(X, np.zeros((N, k)), m.components_, tol=m.tol, update_h=False)[0]
    assert np.abs(Wt - Wtr).max() <= 2e-3 * np.abs(Wtr).max()


@pytest.mark.parametrize("tag", list(dc.NMF))
def test_nmf_default_init_reaches_sklearn_error(cuda, tag):
    N, d, k, seed = dc.NMF[tag]
    X, _, _ = dc.nmf_mixture(N, d, k, seed)
    m = stat.NMF(k, random_state=seed).fit(X)
    # the exact top-k SVD (sklearn: randomized) starts NNDSVDa elsewhere: the same error within 3 %
    assert m.reconstruction_err_ <= 1.03 * float(SK[f"nmf/{tag}/default_err"])
    again = stat.NMF(k, random_state=seed).fit(X)
    assert np.array_equal(m.components_, again.components_)
    assert m.reconstruction_err_ == again.reconstruction_err_
    r = stat.NMF(k, init="random", random_state=seed, max_iter=50).fit(X)
    assert r.components_.min() >= 0 and np.isfinite(r.reconstruction_err_)


@pytest.mark.parametrize("tag", list(dc.ICA))
def test_fastica_matches_sklearn(cuda, tag):
    N, d, seed = dc.ICA[tag]
    X = dc.ica_mixture(N, d, seed)
    ica = stat.FastICA(dc.ICA_K, random_state=seed)
    S = ica.fit_transform(X)
    pre = f"ica/{tag}/"
    assert abs(ica.n_iter_ - int(SK[pre + "n_iter"])) <= 1
    C = SK[pre + "components"]
    np.testing.assert_allclose(ica.components_, C, rtol=0, atol=1e-4 * np.abs(C).max())
    M = SK[pre + "mixing"]
    np.testing.assert_allclose(ica.mixing_, M, rtol=0, atol=1e-4 * np.abs(M).max())
    np.testing.assert_allclose(S, SK[pre + "sources"], rtol=0, atol=1e-3)
    np.testing.assert_allclose(ica.transform(X), S, rtol=0, atol=1e-6)
    again = stat.FastICA(dc.ICA_K, random_state=seed).fit(X)
    assert np.array_equal(again.components_, ica.components_)


def test_wide_stack_n_below_d(cuda):
    """N < d through every estimator: the Gram of the samples, vectors by weighted row sums"""
    X = dc.movie_stack(32, 3, 6)                       # 216 x 3072
    p = stat.PCA(4).fit(X)
    np.testing.assert_allclose(np.linalg.norm(p.components_, axis=1), 1.0, rtol=1e-5)
    ica = stat.FastICA(3, random_state=0).fit(X)
    assert np.all(np.isfinite(ica.components_))
    n = stat.NMF(3, random_state=0, max_iter=30).fit(np.abs(X))
    assert np.isfinite(n.reconstruction_err_)
