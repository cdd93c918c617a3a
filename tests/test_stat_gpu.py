"""atomai_b200.stat on the GPU: the kernels of csrc/stat.cu against the float64 restatement
(oracle/gmm_ref.py), determinism, k-means++ seeding, parity of GaussianMixture / KMeans with sklearn
from identical starts (tests/golden/stat_sklearn.npz) and imlocal against the reference's outputs
(tests/golden/stat_separated.npz)."""
import os

import numpy as np
import pytest
import torch

import stat_cases
from atomai_b200 import ops, stat
from atomai_b200.stat.mixture import _Centred, _kmeans_plusplus
from oracle import gmm_ref

pytestmark = pytest.mark.gpu
HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEP = np.load(os.path.join(HERE, "stat_separated.npz"))
SK = np.load(os.path.join(HERE, "stat_sklearn.npz"))

# (N, d, K): every N, d and K of the issue at least once, with an empty component where K > N / 2
KERNEL_CASES = [(1, 49, 1), (63, 50, 2), (63, 49, 64), (4097, 768, 5), (4097, 50, 17),
                (2 ** 17 + 3, 49, 5), (4097, 3072, 64), (2 ** 17 + 3, 50, 17)]


def _data(N, d, K, seed=0):
    rs = np.random.RandomState(seed)
    centres = rs.randn(K, d) * 2
    X = (centres[rs.randint(0, K, N)] + rs.randn(N, d)).astype(np.float32) + 5.0
    return X


def _centred(X):
    data = _Centred(torch.from_numpy(X).cuda())
    mu = data.mu.cpu().numpy().astype(np.float64)
    return data, X.astype(np.float64) - mu


EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(params=["fp32", "tf32x3"])
def math(request, cuda):
    """the E- / M-step kernels under exact FFMA and on wgmma with split operands"""
    import atomai_b200 as ab
    prev = ab.get_math()
    ab.set_math(request.param)
    yield request.param
    ab.set_math(prev.split("+")[0])


def _dot_tol(d, mag):
    """bound on the fp32 (or split-TF32 tensor-core) evaluation of a d-term dot product whose terms
    have magnitudes summing to `mag`: 8 sqrt(d) eps per unit of magnitude"""
    return 8 * np.sqrt(d) * EPS32 * mag


@pytest.mark.parametrize("N,d,K", KERNEL_CASES)
def test_lloyd_step_matches_float64(math, N, d, K):
    cuda = torch.device("cuda:0")
    X = _data(N, d, K)
    data, Xc = _centred(X)
    rs = np.random.RandomState(1)
    C = (Xc[rs.randint(0, N, K)] + 0.1 * rs.randn(K, d)).astype(np.float32)
    live = K if K == 1 else K - 1
    if K > 1:
        C[-1] += 1e3                                   # an empty cluster
    Cd = torch.from_numpy(C).cuda()
    A, cst = torch.empty(K, d, device=cuda), torch.empty(K, device=cuda)
    ops.stat_kmeans_centres(Cd, A, cst)
    labels = torch.full((N,), -1, dtype=torch.int32, device=cuda)
    dist = torch.empty(N, device=cuda)
    out = torch.empty(1, dtype=torch.float64, device=cuda)
    ch = torch.zeros(1, dtype=torch.float64, device=cuda)
    ops.stat_estep(data.X, data.mu, ops.STAT_KMEANS, A, None, cst, out, labels=labels, rowval=dist,
                   changes=ch)
    got = labels.cpu().numpy()
    d2 = gmm_ref.sqdist(Xc, C)
    lab = d2.argmin(1)
    dmin = d2[np.arange(N), lab]
    # per row: magnitude of ||x||^2 - 2 x.c + ||c||^2 over the live centres only
    C64 = C[:live].astype(np.float64)
    mag = ((Xc ** 2).sum(1)[:, None] + 2 * np.abs(Xc) @ np.abs(C64).T + (C64 ** 2).sum(1)).max(1)
    tol = _dot_tol(d, mag)
    assert np.all(got < live)
    assert np.all(d2[np.arange(N), got] - dmin <= 2 * tol), "label off by more than the rounding"
    assert np.mean(got != lab) <= 0.02
    assert ch.item() == N
    assert np.all(np.abs(dist.cpu().numpy() - dmin) <= 2 * tol)
    assert abs(out.item() - dmin.sum()) <= 2 * tol.sum()
    # the centre sums for the labels the kernel chose
    sx = torch.empty(K, d, dtype=torch.float64, device=cuda)
    nk = torch.empty(K, dtype=torch.float64, device=cuda)
    ops.stat_accum(data.X, data.mu, K, sx, nk=nk, labels=labels)
    onehot = np.eye(K)[got]
    np.testing.assert_array_equal(nk.cpu().numpy(), onehot.sum(0))
    assert np.all(np.abs(sx.cpu().numpy() - onehot.T @ Xc) <= 5e-5 * (onehot.T @ np.abs(Xc)) + 1e-9)


@pytest.mark.parametrize("cov", ["diag", "spherical"])
@pytest.mark.parametrize("N,d,K", KERNEL_CASES)
def test_em_step_matches_float64(math, N, d, K, cov):
    if N * d * K > 2 ** 31:
        pytest.skip("float64 reference too large")
    cuda = torch.device("cuda:0")
    X = _data(N, d, K, seed=2)
    data, Xc = _centred(X)
    rs = np.random.RandomState(3)
    init = rs.randint(0, K, N).astype(np.int32)
    if K > 1:
        init[init == K - 1] = 0                       # component K-1 starts empty
    sx = torch.empty(K, d, dtype=torch.float64, device=cuda)
    sxx, nk = torch.empty_like(sx), torch.empty(K, dtype=torch.float64, device=cuda)
    sph = cov == "spherical"
    means, covs = torch.empty(K, d, device=cuda), torch.empty(K if sph else (K, d), device=cuda)
    weights, cst = torch.empty(K, device=cuda), torch.empty(K, device=cuda)
    A, B = torch.empty(K, d, device=cuda), torch.empty(K, d, device=cuda)
    params = (means, covs, weights, A, B, cst)
    ops.stat_accum(data.X, data.mu, K, sx, sxx, nk, labels=torch.from_numpy(init).cuda())
    onehot = np.eye(K)[init]
    np.testing.assert_array_equal(nk.cpu().numpy(), onehot.sum(0))
    absx = onehot.T @ np.abs(Xc)
    assert np.all(np.abs(sx.cpu().numpy() - onehot.T @ Xc) <= 5e-5 * absx + 1e-9)
    assert np.all(np.abs(sxx.cpu().numpy() - onehot.T @ Xc ** 2) <= 5e-5 * (onehot.T @ Xc ** 2) + 1e-9)
    ops.stat_gmm_params(sx, sxx, nk, N, sph, 1e-6, 1, *params)
    rm, rc, rw = gmm_ref.m_step(Xc, onehot, 1e-6, cov, init=True)
    np.testing.assert_allclose(means.cpu().numpy(), rm, rtol=0, atol=1e-5 * (1 + np.abs(rm).max()))
    # a one-member component's variance is reg_covar after cancelling x^2 against the mean^2
    np.testing.assert_allclose(covs.cpu().numpy(), rc, rtol=1e-4, atol=2e-7 * (Xc ** 2).max())
    np.testing.assert_allclose(weights.cpu().numpy(), rw, rtol=1e-6)
    resp = torch.empty(N, K, device=cuda)
    out = torch.empty(1, dtype=torch.float64, device=cuda)
    ops.stat_estep(data.X, data.mu, ops.STAT_GMM, A, B, cst, out, resp=resp)
    lw = gmm_ref.log_gauss(Xc, means.cpu().numpy(), covs.cpu().numpy(), weights.cpu().numpy())
    rresp, lpn = gmm_ref.e_step(Xc, means.cpu().numpy(), covs.cpu().numpy(), weights.cpu().numpy())
    # per (row, component): magnitude of the terms of sum_j A x + B x^2 + cst in fp32
    Ah, Bh, ch = (t.double().cpu().numpy() for t in (A, B, cst))
    tol_nk = _dot_tol(d, np.abs(Xc) @ np.abs(Ah).T + Xc ** 2 @ np.abs(Bh).T + np.abs(ch)[None])
    # the rows' bound over the components that carry weight (not the reg_covar-only empty one)
    delta = np.where(rresp > 1e-12, tol_nk, 0).max(1)
    got = resp.cpu().numpy()
    assert np.all(np.abs(got - rresp) <= 3 * delta[:, None] + 1e-5)
    top2 = np.sort(lw, 1)[:, -2:] if K > 1 else np.stack([lw[:, 0] - np.inf, lw[:, 0]], 1)
    clear = top2[:, 1] - top2[:, 0] > 2 * delta + 20
    assert np.array_equal(got[clear].argmax(1), lw[clear].argmax(1))
    assert abs(out.item() - lpn.sum()) <= delta.sum() + 1e-6 * N
    ops.stat_accum(data.X, data.mu, K, sx, sxx, nk, resp=resp)
    r64 = resp.double().cpu().numpy()
    np.testing.assert_allclose(nk.cpu().numpy(), r64.sum(0), rtol=5e-5, atol=1e-6)
    # fp32 row sums over 4096-row chunks, bounded relative to the sum of magnitudes; the tensor
    # core's fp32 accumulation truncates instead of rounding, so tf32x3 gets a wider bound
    rel = 5e-5 if math == "fp32" else 2e-4
    for got_s, ref_s, mag in ((sx, r64.T @ Xc, r64.T @ np.abs(Xc)),
                              (sxx, r64.T @ Xc ** 2, r64.T @ Xc ** 2)):
        ratio = (np.abs(got_s.cpu().numpy() - ref_s) / (mag + 1e-30)).max()
        assert ratio <= rel, ratio


def test_fit_is_bit_reproducible_and_row_order_free(cuda):
    X = stat_cases.overlapping(5000, 75, 6, 5)
    fits = [stat.GaussianMixture(6, covariance_type="diag", random_state=0).fit(X) for _ in range(2)]
    for a in ("means_", "covariances_", "weights_"):
        assert np.array_equal(getattr(fits[0], a), getattr(fits[1], a)), a
    assert fits[0].lower_bounds_ == fits[1].lower_bounds_
    lab = fits[0].predict(X)
    perm = np.random.RandomState(0).permutation(len(X))
    g = stat.GaussianMixture(6, covariance_type="diag", init_labels=lab[perm]).fit(X[perm])
    h = stat.GaussianMixture(6, covariance_type="diag", init_labels=lab).fit(X)
    inv = np.argsort(perm)
    assert np.array_equal(g.predict(X[perm])[inv], h.predict(X))
    np.testing.assert_allclose(g.means_, h.means_, atol=1e-5)


def test_kmeans_plusplus_deterministic_and_potential(cuda):
    rs = np.random.RandomState(7)
    X = (rs.randn(600, 10) + 8 * rs.randint(0, 5, (600, 1))).astype(np.float32)
    data = _Centred(torch.from_numpy(X).cuda())
    c1 = _kmeans_plusplus(data, 5, 11).cpu().numpy()
    c2 = _kmeans_plusplus(data, 5, 11).cpu().numpy()
    assert np.array_equal(c1, c2)
    assert not np.array_equal(c1, _kmeans_plusplus(data, 5, 12).cpu().numpy())
    Xc = X - data.mu.cpu().numpy()
    # every seed is a data row
    assert all(np.abs(Xc - c).max(1).min() < 1e-5 for c in c1)
    pot = gmm_ref.sqdist(Xc, c1).min(1).sum()
    # brute force over many uniform seedings: greedy k-means++ lands near the best of them
    best = min(gmm_ref.sqdist(Xc, Xc[np.random.RandomState(s).choice(600, 5, replace=False)])
               .min(1).sum() for s in range(200))
    assert pot <= 8 * (np.log(5) + 2) * best


@pytest.mark.parametrize("tag", list(stat_cases.OVERLAP))
@pytest.mark.parametrize("cov", ["diag", "spherical"])
def test_gaussian_mixture_matches_sklearn(cuda, tag, cov):
    N, d, K, seed = stat_cases.OVERLAP[tag]
    X = stat_cases.overlapping(N, d, K, seed)
    p = f"{tag}/{cov}/"
    g = stat.GaussianMixture(K, covariance_type=cov, random_state=seed,
                             init_labels=SK[f"{tag}/km_labels"])
    lab = g.fit_predict(X)
    lbs = SK[p + "lower_bounds"]
    # float32 scale of the lower bound: sklearn and these kernels each round the fp32 sums over d
    tol = 1e-5 * d * max(1.0, abs(lbs[-1]) / d)
    n = min(len(lbs), len(g.lower_bounds_))
    np.testing.assert_allclose(g.lower_bounds_[:n], lbs[:n], rtol=0, atol=tol)
    if g.n_iter_ != int(SK[p + "n_iter"]):
        assert abs(abs(lbs[-1] - lbs[-2]) - g.tol) <= tol
    # a row may take the other label only where the fitted model's top two weighted log-densities
    # tie within the float32 rounding of the d-term scores
    off = lab != SK[p + "labels"]
    if off.any():
        lw = np.sort(gmm_ref.log_gauss(X[off], g.means_, g.covariances_, g.weights_), 1)
        assert np.all(lw[:, -1] - lw[:, -2] <= 1e-5 * np.abs(lw[:, -1]) + 1e-3)
    np.testing.assert_allclose(g.means_, SK[p + "means"], rtol=0, atol=2e-4)
    np.testing.assert_allclose(g.covariances_, SK[p + "covariances"], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(g.weights_, SK[p + "weights"], rtol=0, atol=1e-5)


@pytest.mark.parametrize("tag", list(stat_cases.OVERLAP))
def test_kmeans_matches_sklearn_lloyd(cuda, tag):
    N, d, K, seed = stat_cases.OVERLAP[tag]
    X = stat_cases.overlapping(N, d, K, seed)
    km = stat.KMeans(K, init=stat_cases.lloyd_init(X, K, seed), n_init=1).fit(X)
    assert np.array_equal(km.labels_, SK[f"{tag}/lloyd_labels"])
    assert km.n_iter_ == int(SK[f"{tag}/lloyd_n_iter"])
    np.testing.assert_allclose(km.cluster_centers_, SK[f"{tag}/lloyd_centres"], rtol=0, atol=1e-5)
    assert np.array_equal(km.predict(X), km.labels_)


def _relabel(got, ref):
    """the permutation p with p[got] == ref (asserting one exists)"""
    pairs = set(zip(got.tolist(), ref.tolist()))
    p = dict(pairs)
    assert len(p) == len(pairs) and len(set(p.values())) == len(p), "not one permutation"
    return p


@pytest.mark.parametrize("tag", list(stat_cases.SEPARATED))
@pytest.mark.parametrize("on_device", [False, True])
def test_imlocal_matches_reference(cuda, tag, on_device):
    w, c, frames = stat_cases.SEPARATED[tag]
    imgs, coords = stat_cases.separated_movie(w, c, frames)
    s = stat.imlocal(torch.from_numpy(imgs).cuda() if on_device else imgs, coords, w, 0)
    assert isinstance(s.imgstack, np.ndarray) and s.imgstack.shape[1:] == (w, w, c)
    cla, cl_all, com_frames = s.gmm(3)
    ref_cf = SEP[f"{tag}/com_frames"]
    p = _relabel(com_frames[:, 2].astype(int), ref_cf[:, 2].astype(int))
    np.testing.assert_array_equal(com_frames[:, [0, 1, 3]], ref_cf[:, [0, 1, 3]])
    for k, v in p.items():
        np.testing.assert_allclose(cla[k - 1], SEP[f"{tag}/cla"][v - 1], rtol=0, atol=1e-6)
        assert len(cl_all[k - 1]) == SEP[f"{tag}/counts"][v - 1]
    if frames > 1:
        d = s.transition_matrix(3, rmax=5, sum_all_transitions=True)
        assert len(d["trajectories"]) == int(SEP[f"{tag}/ntraj"])
        perm = np.array([p[k] for k in (1, 2, 3)]) - 1
        for i, (tr, fr) in enumerate(zip(d["trajectories"], d["frames"])):
            rt = SEP[f"{tag}/traj{i}"]
            np.testing.assert_array_equal(fr, SEP[f"{tag}/frames{i}"])
            np.testing.assert_array_equal(tr[:, :2], rt[:, :2])
            np.testing.assert_array_equal([p[int(k)] for k in tr[:, 2]], rt[:, 2])
        full = np.zeros((3, 3))
        full[np.ix_(perm, perm)] = d["all_transitions"]
        np.testing.assert_allclose(full, SEP[f"{tag}/all_transitions"], rtol=1e-12)


def test_update_classes_gmm_local_runs(cuda):
    imgs, coords = stat_cases.separated_movie(16, 1, 1)
    out = stat.update_classes(coords[0], imgs[0, ..., 0], method="gmm_local", n_components=3,
                              window_size=16)
    assert set(np.unique(out[0][:, -1])) <= {0.0, 1.0, 2.0}
    assert len(out[0]) == 36
    km = stat.update_classes(coords[0], imgs[0, ..., 0], method="kmeans", n_components=3)
    assert km[0].shape == coords[0].shape
