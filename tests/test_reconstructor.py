"""Reconstructor, CPU side: the GP input utilities against goldens made by the unmodified reference
(tests/golden/gp_input.npz, make_golden_gpr.py), the gpytorch parametrisation restated by
CustomGPModel, the argument errors, and the float64 exact-GP oracle (oracle/gpr_ref.py) against
finite differences."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import golden_utils as gu
from oracle import gpr_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAGS = ["5x7", "8x8", "9x4", "1x6", "3x4x5"]


@pytest.mark.parametrize("tag", TAGS)
def test_prepare_gp_input_matches_reference(tag):
    from atomai_b200.utils import prepare_gp_input
    g = gu.load("gp_input.npz")
    x, y, full = prepare_gp_input(g[f"{tag}/image"])
    for got, key in ((x, "x"), (y, "y"), (full, "full")):
        ref = g[f"{tag}/{key}"]
        assert got.dtype == ref.dtype and got.shape == ref.shape
        assert np.array_equal(got, ref)


def test_full_grid_is_row_major_for_images():
    from atomai_b200.utils import prepare_gp_input
    _, _, full = prepare_gp_input(np.ones((3, 5)))
    assert np.array_equal(full, np.indices((3, 5)).reshape(2, -1).T)


@pytest.mark.parametrize("tag", TAGS)
def test_lengthscale_constraints_match_reference(tag):
    from atomai_b200.utils import get_lengthscale_constraints
    g = gu.load("gp_input.npz")
    lo, hi = get_lengthscale_constraints(g[f"{tag}/full"])
    assert lo == g[f"{tag}/lower"].tolist() and hi == g[f"{tag}/upper"].tolist()
    assert [type(v) for v in hi] == [type(v) for v in g[f"{tag}/upper"].tolist()]


def test_create_batches():
    from atomai_b200.utils import create_batches
    a = np.arange(10)
    assert [b.tolist() for b in create_batches(a, 4)] == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
    assert len(create_batches(torch.zeros(8, 2), 8)) == 1
    assert create_batches(a[:0], 3) == []


def _model(d=2, **kw):
    from atomai_b200.nets.gp import CustomGPModel
    return CustomGPModel(torch.rand(7, d), torch.rand(7), None, **kw)


def test_initial_hyperparameters():
    m = _model()
    np.testing.assert_allclose(m.lengthscale.detach().numpy(), np.log(2.0) * np.ones((1, 2)))
    assert float(m.outputscale) == pytest.approx(np.log(2.0))
    assert float(m.noise) == pytest.approx(np.log(2.0) + 1e-4)
    assert float(m.constant) == 0.0


def test_interval_transform_and_initial_value():
    lo, hi = [1.0, 2.0], [5.0, 30.0]
    m = _model(lengthscale_constraints=[lo, hi])
    # an Interval without an initial value leaves raw = 0: the lengthscale starts at the midpoint
    np.testing.assert_allclose(m.lengthscale.detach().numpy()[0], [3.0, 16.0], rtol=1e-6)
    raw = np.array([[-2.5, 1.25]], np.float32)
    m.raw_lengthscale.data = torch.from_numpy(raw)
    want = np.array(lo) + (np.array(hi) - np.array(lo)) / (1 + np.exp(-raw[0].astype(np.float64)))
    np.testing.assert_allclose(m.lengthscale.detach().numpy()[0], want, rtol=1e-6)
    np.testing.assert_allclose(gpr_ref.hyper(dict(ls=raw[0], os=0, noise=0, c=0), (lo, hi))["ls"],
                               want)
    with pytest.raises(ValueError, match="empty intervals"):
        _model(lengthscale_constraints=[[1.0, 3.0], [1.0, 4.0]])


def test_argument_errors():
    from atomai_b200.models import Reconstructor
    X, y = np.random.rand(10, 2), np.random.rand(10)
    with pytest.raises(ValueError, match=re.escape(
            "base_kernel must be either 'rbf', 'matern', or a custom gpytorch.kernels.Kernel "
            "object")):
        Reconstructor(device="cpu").fit(X, y, 1, base_kernel="periodic")
    with pytest.raises(ValueError, match=re.escape(
            "Invalid kernel_type: ski. Supported values are 'sparse' and 'kissgp'.")):
        Reconstructor(device="cpu").fit(X, y, 1, kernel_type="ski")
    with pytest.raises(NotImplementedError):
        Reconstructor(device="cpu").fit(X, y, 1, kernel_type="sparse")
    with pytest.raises(NotImplementedError):
        Reconstructor(device="cpu").fit(X, y, 1, inducing_points=torch.zeros(4, 2))
    with pytest.raises(NotImplementedError):
        Reconstructor(device="cpu").fit(X, y, 1, base_kernel=torch.nn.Identity())
    with pytest.raises(NotImplementedError):
        Reconstructor(device="cpu").fit(np.random.rand(10, 5), y, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        Reconstructor(device="cpu").fit(X, y, 1)


def test_public_surface():
    import atomai_b200 as ab
    from atomai_b200.models.dklgp import Reconstructor
    assert ab.models.Reconstructor is Reconstructor
    for name in ("fit", "predict", "reconstruct"):
        assert callable(getattr(Reconstructor, name))


def _data(n=40, d=2, seed=0):
    rs = np.random.RandomState(seed)
    x = rs.randint(0, 12, size=(n, d)).astype(np.float64) + rs.rand(n, d)
    return x, np.sin(x[:, 0] / 2.0) + 0.1 * rs.randn(n) + 0.5


@pytest.mark.parametrize("kind", ["rbf", "matern"])
@pytest.mark.parametrize("bounded", [False, True])
def test_oracle_gradient_matches_finite_differences(kind, bounded):
    x, y = _data()
    bounds = ([1.0, 1.0], [7.0, 7.0]) if bounded else None
    raw = dict(ls=np.array([0.3, -0.4]), os=0.2, noise=-1.0, c=0.4)
    g = gpr_ref.raw_grad(x, y, raw, kind, bounds)
    h = 1e-6
    for k in gpr_ref.RAW_KEYS:
        for i in range(np.size(raw[k])):
            rp = {kk: np.array(vv, np.float64) for kk, vv in raw.items()}
            rm = {kk: np.array(vv, np.float64) for kk, vv in raw.items()}
            if k == "ls":
                rp[k][i] += h
                rm[k][i] -= h
            else:
                rp[k] = rp[k] + h
                rm[k] = rm[k] - h
            fd = (gpr_ref.neg_mll(x, y, gpr_ref.hyper(rp, bounds), kind) -
                  gpr_ref.neg_mll(x, y, gpr_ref.hyper(rm, bounds), kind)) / (2 * h)
            got = g[k][i] if k == "ls" else g[k]
            assert abs(got - fd) <= 1e-7 + 1e-6 * abs(fd), (k, i, got, fd)


@pytest.mark.parametrize("kind", ["rbf", "matern"])
def test_oracle_posterior_mean_interpolates_at_low_noise(kind):
    x, y = _data(n=25, seed=3)
    p = dict(ls=np.array([1.5, 2.0]), os=1.0, noise=1e-8, c=0.3)
    np.testing.assert_allclose(gpr_ref.posterior_mean(x, y, p, x, kind), y, atol=1e-5)


def test_gpr_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-c", "-Xptxas", "-v", os.path.join(ROOT, "atomai_b200", "csrc", "gpr.cu"),
                        "-o", str(tmp_path / "gpr.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    # d = 1..4 x {RBF, Matern-2.5} x {gram_matvec, gram_f64, gram_f64_adjoint}
    assert len(kernels) == 24, kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) >= len(kernels)
    assert all(a == "0" and b == "0" for a, b in spills), r.stderr
