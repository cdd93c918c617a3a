"""Reconstructor on the GPU: the fused Gram-times-vector kernel (atomai_b200_gram_matvec) against
float64, its run-to-run and batching invariance, the Matern-2.5 Gram adjoint, the exact-GP loss and
gradients, five Adam steps and a whole reconstruction against the float64 oracle
(oracle/gpr_ref.py)."""
import numpy as np
import pytest
import torch

from oracle import gpr_ref

pytestmark = pytest.mark.gpu

U = 2.0 ** -24      # fp32 unit roundoff


def matvec_bound(d):
    """Per-term bound |k_fp32 - k| / u.  t_k = fl(fl(xq - x) * fl(1 / ls)) carries <= 3u relative
    error, r^2 = sum t_k^2 by an fma chain <= (d + 7)u; RBF: |dk/dr^2| r^2 = (r^2/2) e^(-r^2/2)
    <= e^-1, Matern: (5/6)(1 + s) e^-s r^2 <= 0.31; expf / sqrtf / the Matern polynomial add <= 8u.
    The float64 sum adds n 2^-53 relative, negligible here."""
    return (d + 7) / 2.0 + 8.0


def _matvec(xq, x, ls, alpha, c, os_, kind):
    import atomai_b200.ops as ops
    dev = torch.device("cuda:0")
    out = torch.empty(len(xq), device=dev, dtype=torch.float64)
    ops.gram_matvec(torch.from_numpy(xq).to(dev), torch.from_numpy(x).to(dev),
                    (1.0 / torch.from_numpy(ls)).to(torch.float32).to(dev).contiguous(),
                    torch.from_numpy(alpha).to(dev), c, os_, {"rbf": 0, "matern": 1}[kind], out)
    return out.cpu().numpy()


def _points(n, d, rs, scale=40.0):
    return (rs.rand(n, d) * scale).astype(np.float32)


@pytest.mark.parametrize("kind", ["rbf", "matern"])
@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("nq,n", [(1, 1), (1, 3001), (257, 1), (1000, 2500), (3001, 5003)])
def test_gram_matvec_matches_float64(cuda, kind, d, nq, n):
    rs = np.random.RandomState(nq * 7 + n + d)
    xq, x = _points(nq, d, rs), _points(n, d, rs)
    ls = rs.uniform(2.0, 9.0, d)                       # ARD lengthscales
    alpha = rs.randn(n)
    c, os_ = 0.37, 1.7
    got = _matvec(xq, x, ls, alpha, c, os_, kind)
    ref = c + gpr_ref.kernel(xq.astype(np.float64), x.astype(np.float64), ls, os_, kind) @ alpha
    bound = matvec_bound(d) * U * os_ * np.abs(alpha).sum() + 1e-15 * abs(c)
    err = np.abs(got - ref).max()
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("kind", ["rbf", "matern"])
def test_gram_matvec_bit_identical_on_repeat_and_batching(cuda, kind):
    rs = np.random.RandomState(11)
    xq, x = _points(20000, 2, rs, 100.0), _points(4100, 2, rs, 100.0)
    ls, alpha = np.array([3.0, 5.0]), rs.randn(4100)
    a = _matvec(xq, x, ls, alpha, 0.1, 1.3, kind)
    b = _matvec(xq, x, ls, alpha, 0.1, 1.3, kind)
    assert np.array_equal(a, b)
    # small batches split the training points over several CTAs (ordered slots); the sums are
    # the same additions in the same order
    parts = np.concatenate([_matvec(xq[i:i + 777], x, ls, alpha, 0.1, 1.3, kind)
                            for i in range(0, len(xq), 777)])
    assert np.array_equal(a, parts)


def test_gram_matvec_unsplit_launch_matches_split(cuda):
    # 8192 query blocks of 256: more than four waves of CTAs, so one CTA column covers all the
    # training points (no ordered slots)
    rs = np.random.RandomState(12)
    xq, x = _points(1 << 21, 2, rs, 300.0), _points(1500, 2, rs, 300.0)
    ls, alpha = np.array([4.0, 6.0]), rs.randn(1500)
    whole = _matvec(xq, x, ls, alpha, 0.0, 1.0, "matern")
    sub = np.concatenate([_matvec(xq[i:i + 4096], x, ls, alpha, 0.0, 1.0, "matern")
                          for i in range(0, 5 * 4096, 4096)])
    assert np.array_equal(whole[:len(sub)], sub)


@pytest.mark.parametrize("nq,n", [
    (1_050_000, 2000),   # 4102 query blocks: more than the ordered workspace's 4096 ticket groups
    (524_288, 5000),     # 2048 query blocks x 5 chunks: split in 3 CTAs of 2 chunks each
])
def test_gram_matvec_large_launches_match_small_batches(cuda, nq, n):
    rs = np.random.RandomState(nq % 1000 + n)
    xq, x = _points(nq, 2, rs, 1000.0), _points(n, 2, rs, 1000.0)
    ls, alpha = np.array([5.0, 8.0]), rs.randn(n)
    whole = _matvec(xq, x, ls, alpha, 0.2, 1.1, "rbf")
    idx = np.concatenate([np.arange(3000), np.arange(nq - 3000, nq)])
    # batches of 777 queries: 4 query blocks, every chunk in its own CTA (cpc = 1)
    sub = np.concatenate([_matvec(xq[idx[i:i + 777]], x, ls, alpha, 0.2, 1.1, "rbf")
                          for i in range(0, len(idx), 777)])
    assert np.array_equal(whole[idx], sub)
    ref = 0.2 + gpr_ref.kernel(xq[idx].astype(np.float64), x.astype(np.float64), ls, 1.1, "rbf") @ alpha
    assert np.abs(sub - ref).max() <= matvec_bound(2) * U * 1.1 * np.abs(alpha).sum()


def test_gram_matvec_rejects_bad_arguments(cuda):
    from atomai_b200 import _C
    lib = _C.lib()
    assert lib.atomai_b200_gram_matvec(None, None, None, None, 0.0, 1.0, 4, 4, 5, 0, None, None) != 0
    assert b"gram_matvec" in lib.atomai_b200_last_error()
    assert lib.atomai_b200_gram_matvec(None, None, None, None, 0.0, 1.0, 4, 4, 2, 3, None, None) != 0


def test_matern_adjoint_matches_oracle(cuda):
    import atomai_b200.ops as ops
    from atomai_b200.nets.gp import dense_kernel
    rs = np.random.RandomState(5)
    z1, z2 = rs.randn(300, 2) * 3.0, rs.randn(200, 2) * 3.0
    ls, os_ = np.array([1.7, 2.6]), 1.4
    G = rs.randn(300, 200)
    t = lambda a: torch.tensor(a, dtype=torch.float32, device=cuda)
    z1t = t(z1).requires_grad_(True)
    lst, ost = t(ls).requires_grad_(True), t(os_).requires_grad_(True)
    K = dense_kernel(z1t, t(z2), lst, ost, "matern", ops.MATH_FP32)
    (K * t(G)).sum().backward()
    Kr, dls, dos, dx1 = gpr_ref.kernel_grads(z1, z2, ls, os_, "matern")
    assert np.abs(K.detach().cpu().numpy() - Kr).max() <= 3e-5 * os_
    ref_ls = np.array([(G * g).sum() for g in dls])
    ref_os = (G * dos).sum()
    ref_dz1 = (G[..., None] * dx1).sum(1)
    np.testing.assert_allclose(lst.grad.cpu().numpy(), ref_ls, rtol=1e-3,
                               atol=1e-4 * np.abs(ref_ls).max())
    assert abs(float(ost.grad) - ref_os) <= 1e-4 * abs(ref_os) + 1e-3
    e = np.linalg.norm(z1t.grad.cpu().numpy() - ref_dz1) / np.linalg.norm(ref_dz1)
    assert e <= 1e-3, e


@pytest.mark.parametrize("kind", ["rbf", "matern"])
def test_training_gram_and_adjoint_match_float64(cuda, kind):
    import atomai_b200.ops as ops
    rs = np.random.RandomState(8)
    n = 700
    x = rs.randint(-256, 256, size=(n, 2)).astype(np.float64)      # a 512^2 frame, centred
    ls, os_, noise = np.array([7.0, 11.0]), 1.3, 2e-4
    t = lambda a: torch.tensor(a, dtype=torch.float64, device=cuda)
    K = torch.empty((n, n), device=cuda, dtype=torch.float64)
    ops.gram_f64(t(x), t(1.0 / ls), os_, noise, {"rbf": 0, "matern": 1}[kind], K)
    Kr, dls, dos, _ = gpr_ref.kernel_grads(x, x, ls, os_, kind)
    Kg = K.cpu().numpy()
    assert np.array_equal(Kg, Kg.T)
    assert np.abs(Kg - Kr - noise * np.eye(n)).max() <= 1e-14 * os_
    G = rs.randn(n, n)
    s = torch.empty(4, device=cuda, dtype=torch.float64)
    ops.gram_f64_adjoint(t(x), t(1.0 / ls), {"rbf": 0, "matern": 1}[kind], t(G), s)
    s = s.cpu().numpy()
    ref_ls = np.array([(G * g).sum() for g in dls])
    np.testing.assert_allclose(os_ * s[:2] / ls, ref_ls, rtol=1e-10)
    np.testing.assert_allclose(s[2], (G * dos).sum(), rtol=1e-10)
    np.testing.assert_allclose(s[3], np.trace(G), rtol=1e-12)
    s2 = torch.empty(4, device=cuda, dtype=torch.float64)
    ops.gram_f64_adjoint(t(x), t(1.0 / ls), {"rbf": 0, "matern": 1}[kind], t(G), s2)
    assert np.array_equal(s, s2.cpu().numpy())


def test_low_noise_fit_on_wide_coordinates(cuda):
    """A smooth, almost noiseless scan spread over a 512^2 frame: the float64 Gram stays positive
    definite down to the 1e-4 noise floor, so 100 cycles train without a failed Cholesky."""
    from atomai_b200.models import Reconstructor
    rs = np.random.RandomState(30)
    idx = rs.choice(512 * 512, 1800, replace=False)
    x = np.stack([idx // 512, idx % 512], 1).astype(np.float64)
    y = np.sin(x[:, 0] / 40.0) * np.cos(x[:, 1] / 55.0) + 2.0
    rec = Reconstructor()
    rec.fit(x, y, 100, lengthscale_constraints=[[1.0, 1.0], [257.0, 257.0]], print_loss=1000)
    assert np.all(np.isfinite(rec.train_loss)) and rec.train_loss[-1] < rec.train_loss[0]
    m = rec.gp_model
    with torch.no_grad():
        m.raw_noise.fill_(-30.0)              # noise = softplus(-30) + 1e-4 = the floor
        m._cache = None
        mean = rec.predict(x).cpu().numpy()
    assert np.abs(mean - y).max() < 5e-2


def test_training_step_memory_within_checked_count(cuda):
    from atomai_b200.models import Reconstructor
    from atomai_b200.trainers.gptrainer import _EXACT_GP_NXN
    x, y = _pixels(3000, 100, 31)
    rec = Reconstructor()
    rec.compile_trainer(x, y, 1, base_kernel="matern")
    rec.train_step()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    rec.train_step()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= _EXACT_GP_NXN * 8 * 3000 ** 2, peak / (8 * 3000 ** 2)


def _pixels(n, side, seed):
    rs = np.random.RandomState(seed)
    idx = rs.choice(side * side, n, replace=False)
    x = np.stack([idx // side, idx % side], 1).astype(np.float64)
    y = np.cos(x[:, 0] / 3.0) * np.sin(x[:, 1] / 4.0) + 0.05 * rs.randn(n) + 1.0
    return x, y


def _set_raw(m, raw):
    with torch.no_grad():
        m.raw_lengthscale.copy_(torch.tensor(raw["ls"]).reshape(1, -1))
        m.raw_outputscale.fill_(float(raw["os"]))
        m.raw_noise.fill_(float(raw["noise"]))
        m.raw_constant.fill_(float(raw["c"]))


@pytest.mark.parametrize("kind", ["rbf", "matern"])
@pytest.mark.parametrize("bounded", [False, True])
def test_neg_mll_and_gradients_match_oracle(cuda, kind, bounded):
    from atomai_b200.nets.gp import CustomGPModel
    x, y = _pixels(300, 32, 7)
    bounds = ([1.0, 1.0], [16.0, 16.0]) if bounded else None
    raw = dict(ls=np.array([1.5, 1.0]), os=0.3, noise=-2.0, c=0.8)
    m = CustomGPModel(torch.tensor(x, dtype=torch.float32, device=cuda),
                      torch.tensor(y, device=cuda), None, base_kernel=kind,
                      lengthscale_constraints=bounds).to(cuda)
    _set_raw(m, raw)
    loss = m.neg_mll()
    loss.backward()
    ref = gpr_ref.neg_mll(x, y, gpr_ref.hyper(raw, bounds), kind)
    g = gpr_ref.raw_grad(x, y, raw, kind, bounds)
    # the fp32 Gram forms r^2 by a norm expansion: absolute error ~ u (|a|^2 + |b|^2) ~ 5e-5 for
    # centred 32-pixel coordinates over lengthscales ~ 1.3, carried through the float64 algebra
    assert abs(float(loss.detach()) - ref) <= 1e-4 * abs(ref) + 1e-6
    got = dict(ls=m.raw_lengthscale.grad.cpu().numpy().reshape(-1),
               os=float(m.raw_outputscale.grad), noise=float(m.raw_noise.grad),
               c=float(m.raw_constant.grad))
    for k in gpr_ref.RAW_KEYS:
        np.testing.assert_allclose(got[k], g[k], rtol=5e-3, atol=1e-4, err_msg=k)


@pytest.mark.parametrize("kind", ["rbf", "matern"])
def test_five_adam_steps_match_float64(cuda, kind):
    from atomai_b200.models import Reconstructor
    x, y = _pixels(400, 40, 9)
    bounds = [[1.0, 1.0], [20.0, 20.0]]
    rec = Reconstructor()
    rec.fit(x, y, 5, base_kernel=kind, lengthscale_constraints=bounds, print_loss=100)
    raw, losses = gpr_ref.fit(x, y, 5, 0.1, kind, bounds)
    m = rec.gp_model
    # fp32 raw parameters and Gram: each Adam step of ~lr moves by <= lr * (gradient rel. error)
    np.testing.assert_allclose(rec.train_loss, losses, rtol=2e-4)
    np.testing.assert_allclose(m.raw_lengthscale.detach().cpu().numpy().reshape(-1), raw["ls"],
                               atol=1e-3)
    for name, k in (("raw_outputscale", "os"), ("raw_noise", "noise"), ("raw_constant", "c")):
        assert abs(float(getattr(m, name).detach()) - float(raw[k])) <= 1e-3, name


def lattice_image(side=64, spacing=8, sigma=1.6, keep=0.15, seed=21):
    rs = np.random.RandomState(seed)
    ii, jj = np.mgrid[:side, :side].astype(np.float64)
    img = np.full((side, side), 0.1)
    for ci in np.arange(spacing / 2, side, spacing):
        for cj in np.arange(spacing / 2, side, spacing):
            img += np.exp(-((ii - ci) ** 2 + (jj - cj) ** 2) / (2 * sigma ** 2))
    mask = rs.rand(side, side) < keep
    return img, (img * mask).astype(np.float32)


def test_reconstruct_matches_oracle(cuda):
    from atomai_b200.models import Reconstructor
    full, sparse = lattice_image()
    got = Reconstructor().reconstruct(sparse, training_cycles=30, print_loss=100)
    ref = gpr_ref.reconstruct(sparse, 30)
    assert got.shape == sparse.shape and got.dtype == np.float32
    # fp32 hyper-parameters under Adam against the float64 trajectory; the mean itself is exact to
    # ~1e-6 (test_gram_matvec_matches_float64)
    rng = full.max() - full.min()
    assert np.abs(got - ref).max() <= 5e-3 * rng, np.abs(got - ref).max()


def test_predict_batches_equal_one_batch(cuda):
    from atomai_b200.models import Reconstructor
    from atomai_b200.utils import prepare_gp_input
    _, sparse = lattice_image(seed=22)
    X, y, X_full = prepare_gp_input(sparse)
    rec = Reconstructor()
    rec.fit(X, y, 3, base_kernel="matern", print_loss=100)
    one = rec.predict(X_full)
    parts = rec.predict(X_full, batch_size=1000)
    assert one.shape == (len(X_full),) and one.dtype == torch.float32
    assert torch.equal(one, parts)


def test_exact_gp_memory_is_checked_first(cuda):
    from atomai_b200.models import Reconstructor
    n = 2_000_000                 # float64 N x N = 32 TB
    with pytest.raises(MemoryError, match="N = 2000000"):
        Reconstructor().fit(np.random.rand(n, 2), np.random.rand(n), 1)
