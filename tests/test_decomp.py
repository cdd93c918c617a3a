"""atomai_b200.stat PCA / NMF / FastICA without a GPU: the float64 restatement (oracle/decomp_ref.py),
iterated from the goldens' starting points, reproduces sklearn's NMF and FastICA results
(tests/golden/decomp_sklearn.npz); the host-side initialisations equal sklearn's and the oracle's;
every argument error is raised before a device is touched."""
import inspect
import os

import numpy as np
import pytest
import torch

import decomp_cases as dc
from atomai_b200 import stat
from atomai_b200.stat import decomposition
from oracle import decomp_ref

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SK = np.load(os.path.join(HERE, "decomp_sklearn.npz"))


@pytest.mark.parametrize("tag", list(dc.NMF))
def test_oracle_nmf_reproduces_sklearn_from_custom_init(tag):
    N, d, k, seed = dc.NMF[tag]
    X, W0, H0 = dc.nmf_mixture(N, d, k, seed)
    W, H, n_iter = decomp_ref.nmf_cd(X, W0, H0, tol=dc.NMF_TOL)
    p = f"nmf/{tag}/"
    assert n_iter == int(SK[p + "n_iter"])
    np.testing.assert_allclose(W, SK[p + "W"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(H, SK[p + "H"], rtol=1e-9, atol=1e-12)
    err = np.linalg.norm(X.astype(np.float64) - W @ H)
    np.testing.assert_allclose(err, SK[p + "err"], rtol=1e-10)


@pytest.mark.parametrize("tag", list(dc.ICA))
def test_oracle_fastica_reproduces_sklearn(tag):
    N, d, seed = dc.ICA[tag]
    X = dc.ica_mixture(N, d, seed)
    mean, K, X1 = decomp_ref.whitening(X, dc.ICA_K)
    w_init = np.random.RandomState(seed).normal(size=(dc.ICA_K, dc.ICA_K))
    W, n_iter = decomp_ref.ica_par(X1, w_init)
    S = (W @ K @ (X - mean).T).T
    W = W / S.std(0)[:, None]
    p = f"ica/{tag}/"
    assert n_iter == int(SK[p + "n_iter"])
    np.testing.assert_allclose(W @ K, SK[p + "components"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(S / S.std(0), SK[p + "sources"], rtol=1e-7, atol=1e-9)
    # the unit-variance rescale the estimator applies from the whitening identity
    s_std = np.sqrt(np.einsum("ij,ij->i", W * S.std(0)[:, None], W * S.std(0)[:, None]) / N)
    np.testing.assert_allclose(s_std, S.std(0), rtol=1e-9)


def test_oracle_gram_and_sweeps_are_consistent():
    X, W0, H0 = dc.nmf_mixture(40, 30, 3, 5)
    np.testing.assert_allclose(decomp_ref.gram(X, X.mean(0), rows=True).trace(),
                               decomp_ref.gram(X, X.mean(0)).trace(), rtol=1e-12)
    W1, vw, WtW = decomp_ref.nmf_w_sweep(X, W0, H0)
    H1, vh, HHt = decomp_ref.nmf_h_sweep(X, W1, H0)
    W, H, _ = decomp_ref.nmf_cd(X, W0, H0, max_iter=1)
    np.testing.assert_array_equal(W, W1)
    np.testing.assert_array_equal(H, H1)
    np.testing.assert_allclose(WtW, W1.T @ W1)
    np.testing.assert_allclose(HHt, H1 @ H1.T)
    assert vw > 0 and vh > 0


def test_random_init_equals_sklearn_bit_for_bit():
    nmf = pytest.importorskip("sklearn.decomposition._nmf")
    X, _, _ = dc.nmf_mixture(300, 70, 6, 3)
    W, H = decomposition._random_init(X.mean(), 300, 70, 6, 11)
    Ws, Hs = nmf._initialize_nmf(X, 6, init="random", random_state=11)
    assert W.dtype == Ws.dtype == np.float32
    np.testing.assert_array_equal(W, Ws)
    np.testing.assert_array_equal(H, Hs)


@pytest.mark.parametrize("avg", [None, 0.37])
def test_nndsvd_matches_oracle(avg):
    rs = np.random.RandomState(4)
    X = np.abs(rs.randn(50, 20))
    U, S, V = np.linalg.svd(X, full_matrices=False)
    k = 5
    W, H = decomposition._nndsvd(*(torch.from_numpy(np.ascontiguousarray(a))
                                   for a in (U[:, :k], S[:k], V[:k])), avg)
    Wr, Hr = decomp_ref.nndsvd(U[:, :k], S[:k], V[:k], avg)
    np.testing.assert_allclose(W.numpy(), Wr, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(H.numpy(), Hr, rtol=1e-14, atol=1e-15)


def test_parameters_are_sklearns():
    sk = pytest.importorskip("sklearn.decomposition")
    for name in ("PCA", "NMF", "FastICA"):
        ours = inspect.signature(getattr(stat, name)).parameters
        theirs = inspect.signature(getattr(sk, name)).parameters
        for p, v in ours.items():
            assert p in theirs, (name, p)
            if p != "n_components":      # sklearn's NMF default is 'auto' (n_features), ours None
                assert v.default == theirs[p].default, (name, p)
            assert v.kind == theirs[p].kind, (name, p)


X = np.abs(np.random.RandomState(0).randn(10, 4)).astype(np.float32)


@pytest.mark.parametrize("call,exc", [
    (lambda: stat.PCA(0).fit(X), ValueError),
    (lambda: stat.PCA(5).fit(X), ValueError),
    (lambda: stat.PCA(0.9).fit(X), NotImplementedError),
    (lambda: stat.PCA(1).fit(X[:1]), ValueError),
    (lambda: stat.NMF(65).fit(np.ones((100, 70), np.float32)), ValueError),
    (lambda: stat.NMF(0).fit(X), ValueError),
    (lambda: stat.NMF(2, init="bogus").fit(X), ValueError),
    (lambda: stat.NMF(2, init="nndsvdar").fit(X), NotImplementedError),
    (lambda: stat.NMF(5, init="nndsvda").fit(X), ValueError),
    (lambda: stat.NMF(2, max_iter=0).fit(X), ValueError),
    (lambda: stat.NMF(2).fit(-X), ValueError),
    (lambda: stat.NMF(2, init="custom").fit(X), ValueError),
    (lambda: stat.NMF(2, init="custom").fit_transform(X, W=-np.ones((10, 2)), H=np.ones((2, 4))),
     ValueError),
    (lambda: stat.FastICA(2, algorithm="deflation").fit(X), NotImplementedError),
    (lambda: stat.FastICA(2, whiten=False).fit(X), NotImplementedError),
    (lambda: stat.FastICA(2, fun="cube").fit(X), NotImplementedError),
    (lambda: stat.FastICA(65).fit(np.ones((100, 70), np.float32)), ValueError),
    (lambda: stat.FastICA(2, w_init=np.eye(3)).fit(X), ValueError),
    (lambda: stat.FastICA(2).fit(X[:1]), ValueError),
])
def test_argument_errors_raise_before_device(call, exc, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device touched")
    monkeypatch.setattr(decomposition, "_load", no_device)
    with pytest.raises(exc):
        call()
