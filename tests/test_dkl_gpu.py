"""DKL row: native fcFeatureExtractor (forward + backward) against goldens produced by the
unmodified reference (tests/golden/dkl_fe.npz, make_golden_dkl.py), and the dense deep-kernel Gram
against the float64 numpy oracle (oracle/gram_ref.py; gpytorch is not installable here, so the
Gram is pinned to gpytorch's published kernel formulas only — see its header)."""
import numpy as np
import pytest
import torch

import golden_utils as gu
from oracle import gram_ref

pytestmark = pytest.mark.gpu

FE_CASES = {"fe_37_2": dict(feat=37, embedim=2, n=300, seed=900),
            "fe_64_128": dict(feat=64, embedim=128, n=520, seed=910)}
# fp32: exact FFMA GEMMs; tf32x3 / tf32: the MLP runs as 1x1 convolutions on wgmma.
# (forward max-rel, gradient rel-L2).  tf32x3 forward: the tensor core accumulates K = 1000 in
# fp32 with truncation, ~1e-5; tf32 gradients go through three ReLU masks and are only guarded
# against gross errors (same policy as the TF32 VAE tests).
TOL = {"fp32": (1e-5, 2e-4), "tf32x3": (5e-5, 1e-3), "tf32": (3e-3, 3e-1)}


@pytest.mark.parametrize("math", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("tag", list(FE_CASES))
def test_feature_extractor_vs_reference(cuda, tag, math):
    import atomai_b200 as ab
    from collections import OrderedDict
    from atomai_b200.nets import fcFeatureExtractor
    ab.set_math(math)
    c = FE_CASES[tag]
    gold = gu.load("dkl_fe.npz")
    fe = fcFeatureExtractor(c["feat"], c["embedim"])
    assert [n for n, _ in fe.named_children()] == ["linear1", "relu1", "linear2", "relu2",
                                                   "linear3", "relu3", "linear4"]
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in fe.state_dict().items())
    fe.load_state_dict({k: torch.from_numpy(v) for k, v in gu.fill_state_dict(shapes, c["seed"]).items()})
    fe = fe.to(cuda)
    rs = np.random.RandomState(c["seed"] + 1)
    x = torch.from_numpy(rs.randn(c["n"], c["feat"]).astype(np.float32)).to(cuda).requires_grad_(True)
    g = torch.from_numpy(rs.randn(c["n"], c["embedim"]).astype(np.float32)).to(cuda)
    y = fe(x)
    ref = gold[f"{tag}/y"]
    tol_y, tol_g = TOL[math]
    assert np.abs(y.detach().cpu().numpy() - ref).max() <= tol_y * np.abs(ref).max()
    (y * g).sum().backward()
    dx_ref = gold[f"{tag}/dx"]
    assert np.abs(x.grad.cpu().numpy() - dx_ref).max() <= tol_g * np.abs(dx_ref).max()
    for k, p in fe.named_parameters():
        gr = p.grad.detach().cpu().numpy()
        got = gu.sample_flat(gr, 97) if gr.size > 4096 else gr
        r = gold[f"{tag}/grad/{k}"]
        e = np.linalg.norm((got.reshape(-1) - r.reshape(-1)).astype(np.float64))
        n_ = np.linalg.norm(r.reshape(-1).astype(np.float64)) + 1e-30
        assert e <= tol_g * n_, (k, e / n_)
    ab.set_math("tf32x3")


@pytest.mark.parametrize("math", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("kind", ["rbf", "matern"])
def test_dense_gram_matches_oracle(cuda, kind, math):
    import atomai_b200 as ab
    from atomai_b200.nets import dense_gram
    ab.set_math(math)
    rs = np.random.RandomState(0)
    x1 = rs.randn(333, 128).astype(np.float32)      # 333 = 41*8 + 5, 257 = 16*16 + 1: remainders
    x2 = rs.randn(257, 128).astype(np.float32)
    ls = (rs.rand(128) * 4 + 8).astype(np.float32)
    Kd = torch.empty(333, 260, device=cuda)[:, :257]     # row stride % 4 == 0 -> tensor path
    from atomai_b200 import ops, engine
    inv = torch.from_numpy(1.0 / ls).to(cuda)
    ops.gram(torch.from_numpy(x1).to(cuda), torch.from_numpy(x2).to(cuda), inv, 1.7,
             {"rbf": 0, "matern": 1}[kind], Kd, engine._MATH["mode"])
    ref = gram_ref.gram(x1, x2, ls, 1.7, kind)
    tol = 2e-3 if math == "tf32" else 2e-5
    assert np.abs(Kd.cpu().numpy() - ref).max() <= tol * np.abs(ref).max()
    K2 = dense_gram(torch.from_numpy(x1).to(cuda), torch.from_numpy(x2).to(cuda),
                    torch.from_numpy(ls), 1.7, kind).cpu().numpy()
    assert K2.shape == (333, 257) and np.abs(K2 - ref).max() <= tol * np.abs(ref).max()
    ab.set_math("tf32x3")


def test_gram_properties_at_scale(cuda):
    """Size-independent properties on a larger problem: symmetry, unit diagonal, bounds."""
    import atomai_b200 as ab
    from atomai_b200.nets import dense_gram
    ab.set_math("tf32x3")
    x = torch.randn(4096, 128, device=cuda)
    ls = torch.full((128,), 128 ** 0.5)
    K = dense_gram(x, x, ls, 1.0, "rbf")
    assert torch.allclose(K, K.t(), atol=2e-6)
    assert torch.allclose(torch.diagonal(K), torch.ones(4096, device=cuda), atol=1e-5)
    assert float(K.min()) >= 0.0 and float(K.max()) <= 1.0 + 1e-6


def test_dense_rbf_gradients(cuda):
    """Adjoint of the native Gram (w.r.t. both inputs, ARD lengthscales, outputscale) against
    torch autograd of the closed formula in float64."""
    import atomai_b200 as ab
    from atomai_b200.nets import dense_rbf
    ab.set_math("tf32x3")
    torch.manual_seed(0)
    z1 = torch.randn(200, 3, device=cuda, requires_grad=True)
    z2 = torch.randn(120, 3, device=cuda, requires_grad=True)
    ls = (torch.rand(3, device=cuda) + 0.5).requires_grad_(True)
    os_ = torch.tensor(1.3, device=cuda, requires_grad=True)
    G = torch.randn(200, 120, device=cuda)
    (dense_rbf(z1, z2, ls, os_) * G).sum().backward()
    a, b, l, o = (t.detach().cpu().double().requires_grad_(True) for t in (z1, z2, ls, os_))
    d2 = (((a[:, None] - b[None]) / l) ** 2).sum(-1)
    ((o * torch.exp(-0.5 * d2)) * G.cpu().double()).sum().backward()
    for got, ref in ((z1.grad, a.grad), (z2.grad, b.grad), (ls.grad, l.grad), (os_.grad, o.grad)):
        e = (got.cpu().double() - ref).norm() / (ref.norm() + 1e-30)
        assert e <= 1e-4, float(e)


def test_dklgpr_api(cuda):
    """dklGPR with the reference's call patterns (test/models/test_dklgpr.py): fit / predict /
    embed / ensembles / sampling shapes, and the loss goes down."""
    import atomai_b200 as ab
    from atomai_b200.models import dklGPR
    ab.set_math("tf32x3")
    rs = np.random.RandomState(0)
    indim = 32
    X = rs.randn(96, indim)
    w = rs.randn(indim) / indim ** 0.5
    y = np.tanh(X @ w) + 0.05 * rs.randn(96)
    X_test = rs.randn(50, indim)
    t = dklGPR(indim, precision="single")
    assert len(t.train_loss) == 0
    t.fit(X, y, 30, print_loss=100)
    assert len(t.train_loss) == 30 and t.train_loss[-1] < t.train_loss[0]
    mean, var = t.predict(X_test)
    assert mean.shape == (50,) and var.shape == (50,) and np.all(var > 0)
    assert isinstance(mean, np.ndarray) and isinstance(var, np.ndarray)
    mtr, _ = t.predict(X)
    assert np.corrcoef(mtr, y)[0, 1] > 0.8          # it actually regresses
    emb = t.embed(X_test)
    assert emb.shape == (50, 2)
    s = t.sample_from_posterior(X_test, num_samples=7)
    assert s.shape == (7, 1, 50)
    # independent outputs
    y2 = np.stack([y, -y])
    t2 = dklGPR(indim, shared_embedding_space=False, precision="single")
    t2.fit(X, y2, 2)
    m2, v2 = t2.predict(X_test)
    assert m2.shape == (2, 50) and v2.shape == (2, 50)
    assert t2.embed(X_test).shape == (2, 50, 2)
    # ensemble of 3 models on a scalar target
    t3 = dklGPR(indim, precision="single")
    with pytest.warns(UserWarning):
        t3.fit_ensemble(X, y, 2, n_models=3)
    m3, v3 = t3.predict(X_test)
    assert m3.shape == (3, 50) and len(t3.train_loss) == 2
    ts, idx = t3.thompson(X_test)
    assert ts.shape == (3, 50) and idx.shape == (3,)
