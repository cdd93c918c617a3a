"""
Deep-kernel-learning modules (atomai/nets/gp.py:14-60).

  * fcFeatureExtractor — the MLP (feat_dim -> 1000 -> 500 -> 50 -> embedim, ReLU) as an
    nn.Sequential with the reference's module names (`linear1`, `relu1`, ...), executed as a chain
    of native GEMM kernels with fused bias + ReLU epilogues;
  * DeepKernel — feature extractor followed by the dense RBF / Matern-2.5 Gram kernel
    (atomai_b200/csrc/gram.cu): K = os * k(||(f(x1) - f(x2)) / lengthscale||).  The reference never
    forms a dense Gram: it configures gpytorch's KISS-GP (GridInterpolationKernel) around the same
    ScaleKernel(RBFKernel(ard)) (nets/gp.py:41-46).  gpytorch is not vendored by the reference and
    not installed in this image; GPRegressionModel therefore needs gpytorch at call time and the
    dense kernel is exposed for the covariance evaluation itself (SURVEY.md §0.6, §8a a15-a16);
  * CustomGPModel — the Reconstructor's exact GP on the raw inputs (atomai/nets/gp.py:63-128), its
    predictive mean on the fused Gram-times-vector kernel (atomai_b200/csrc/gpr.cu).
"""
from typing import Optional

import torch

from .. import engine, ops
from ..engine import Tape


class fcFeatureExtractor(torch.nn.Sequential):
    """MLP feature extractor (atomai/nets/gp.py:14-26)."""
    def __init__(self, feat_dim, embedim, **kwargs):
        super(fcFeatureExtractor, self).__init__()
        hidden_dim = kwargs.get("hidden_dim")
        hidden_dim = [1000, 500, 50] if hidden_dim is None else list(hidden_dim)
        hidden_dim.append(embedim)
        self.add_module("linear1", torch.nn.Linear(feat_dim, hidden_dim[0]))
        for i, h in enumerate(hidden_dim[1:]):
            self.add_module('relu{}'.format(i+1), torch.nn.ReLU())
            self.add_module('linear{}'.format(i+2), torch.nn.Linear(hidden_dim[i], h))

    def _emit(self, tape: Tape, x):
        mods = list(self.children())
        lins, acts = [], []
        for i, m in enumerate(mods):
            if isinstance(m, torch.nn.Linear):
                relu_next = i + 1 < len(mods) and isinstance(mods[i + 1], torch.nn.ReLU)
                lins.append(m)
                acts.append("relu" if relu_next else None)
        return tape.mlp(x, lins, acts)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.dtype != torch.float32:
            raise NotImplementedError("the native feature extractor computes in fp32 "
                                      "(precision='single'); float64 is not implemented")
        b = x.shape[0]
        y = engine.run_multi(self, self._emit, (x.reshape(b, 1, 1, -1).contiguous(),))
        return y.reshape(b, -1)


def dense_gram(x1: torch.Tensor, x2: torch.Tensor, lengthscale: torch.Tensor,
               outputscale: float = 1.0, kind: str = "rbf", math: Optional[int] = None
               ) -> torch.Tensor:
    """K[i, j] = outputscale * k(||(x1_i - x2_j) / lengthscale||) with gpytorch's RBFKernel /
    MaternKernel(nu=2.5) + ScaleKernel definitions, as one fused tiled kernel (no n1 x n2 distance
    matrix in HBM, exponentiation in the epilogue).  Forward only.  `math` (an ops.MATH_* mode)
    defaults to the library-wide mode of atomai_b200.set_math."""
    assert x1.is_cuda and x1.dtype == torch.float32 and x1.dim() == 2 and x2.dim() == 2
    inv_ls = (1.0 / lengthscale.to(x1.device, torch.float32).reshape(-1)).contiguous()
    if inv_ls.numel() == 1:
        inv_ls = inv_ls.expand(x1.shape[1]).contiguous()
    n2 = x2.shape[0]      # row stride padded to 16 B so that the tensor-core path applies
    out = torch.empty((x1.shape[0], -(-n2 // 4) * 4), device=x1.device, dtype=torch.float32)[:, :n2]
    ops.gram(x1.contiguous(), x2.contiguous(), inv_ls, float(outputscale),
             {"rbf": 0, "matern": 1}[kind], out, engine._MATH["mode"] if math is None else math)
    return out


class DeepKernel(torch.nn.Module):
    """k(x, x') = outputscale * RBF((f(x) - f(x')) / lengthscale) with f = fcFeatureExtractor."""
    def __init__(self, feat_dim: int, embedim: int = 2, kind: str = "rbf", **kwargs):
        super().__init__()
        self.feature_extractor = fcFeatureExtractor(feat_dim, embedim, **kwargs)
        self.raw_lengthscale = torch.nn.Parameter(torch.zeros(embedim))
        self.raw_outputscale = torch.nn.Parameter(torch.zeros(()))
        self.kind = kind

    @property
    def lengthscale(self):
        return torch.nn.functional.softplus(self.raw_lengthscale)

    @property
    def outputscale(self):
        return torch.nn.functional.softplus(self.raw_outputscale)

    def forward(self, x1: torch.Tensor, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
        with torch.no_grad():
            z1 = self.feature_extractor(x1)
            z2 = z1 if x2 is None else self.feature_extractor(x2)
            return dense_gram(z1, z2, self.lengthscale, float(self.outputscale), self.kind)


class _DenseGramFn(torch.autograd.Function):
    """K = outputscale * k(r^2), r^2 = ||(z1 - z2) / ls||^2, with the native Gram kernel forward and
    its adjoint built from the kernel output: with W = dK * (-2 dK/dr^2),
        dz1 = -(rowsum(W) * z1 - W z2) / ls^2        dz2 = -(colsum(W) * z2 - W^T z1) / ls^2
        dls = sum_ij W_ij (z1_i - z2_j)^2 / ls^3      dos = sum(dK * K) / os
    (the two n x n x d products run on the library's own GEMM kernel).  RBF: -2 dK/dr^2 = K.
    Matern-2.5 (s = sqrt(5) r): -2 dK/dr^2 = 5/3 os (1 + s) exp(-s) = 5/3 K (1 + s) / (1 + s + s^2/3),
    with r^2 = -2 log(exp(-r^2 / 2)) from the native RBF Gram at unit outputscale (the factor is 0
    where that underflows, r^2 > ~200, where K / os < e^-31)."""

    @staticmethod
    def forward(ctx, z1, z2, ls, os_, kind="rbf", math=None):
        K = dense_gram(z1, z2, ls.detach(), float(os_), kind, math)
        ctx.save_for_backward(z1, z2, ls, os_, K)
        ctx.kind, ctx.math = kind, math
        return K

    @staticmethod
    def backward(ctx, dK):
        z1, z2, ls, os_, K = ctx.saved_tensors
        if ctx.kind == "rbf":
            W = (dK.to(torch.float32) * K).contiguous()
        else:
            e = dense_gram(z1, z2, ls.detach(), 1.0, "rbf", ctx.math)
            d2 = -2.0 * torch.log(e)
            sr = torch.sqrt(5.0 * d2)
            m = torch.where(e > 0, (5.0 / 3.0) * K * (1.0 + sr) / (1.0 + sr + (5.0 / 3.0) * d2),
                            torch.zeros_like(K))
            W = (dK.to(torch.float32) * m).contiguous()
        n1, n2, d = z1.shape[0], z2.shape[0], z1.shape[1]
        z1c, z2c = z1.contiguous(), z2.contiguous()
        Wz2 = torch.empty((n1, d), device=W.device, dtype=torch.float32)
        Wtz1 = torch.empty((n2, d), device=W.device, dtype=torch.float32)
        ops.gemm(W, n2, 1, z2c, d, 1, Wz2, d, n1, d, n2)            # W @ z2
        ops.gemm(W, 1, n2, z1c, d, 1, Wtz1, d, n2, d, n1)           # W^T @ z1
        rs, cs = W.sum(1, keepdim=True), W.sum(0)[:, None]
        inv2 = 1.0 / (ls * ls)
        dz1 = -(rs * z1c - Wz2) * inv2
        dz2 = -(cs * z2c - Wtz1) * inv2
        s = (rs * z1c * z1c).sum(0) + (cs * z2c * z2c).sum(0) - 2.0 * (z1c * Wz2).sum(0)
        dls = s / (ls * ls * ls)
        dos = (dK * K).sum() / os_
        return dz1, dz2, dls, dos, None, None


def dense_rbf(z1, z2, lengthscale, outputscale):
    """Differentiable dense ScaleKernel(RBFKernel(ard)) Gram on the native kernels."""
    return _DenseGramFn.apply(z1, z2, lengthscale, outputscale)


def dense_kernel(z1, z2, lengthscale, outputscale, kind: str = "rbf", math: Optional[int] = None):
    """Differentiable dense ScaleKernel(RBFKernel | MaternKernel(nu=2.5), ard) Gram on the native
    kernels (`kind` "rbf" | "matern"); `math` as dense_gram."""
    return _DenseGramFn.apply(z1, z2, lengthscale, outputscale, kind, math)


class ScaleToBounds(torch.nn.Module):
    """gpytorch.utils.grid.ScaleToBounds(lower, upper) restated (gpytorch is a third-party
    dependency of the reference, not vendored and not installed here; atomai/nets/gp.py:48,56):
    in training mode rescales by the batch min / max (and remembers them), in eval mode clamps to
    the remembered range; output spans 0.95 * [lower, upper].  Parity with gpytorch UNPINNED."""
    def __init__(self, lower_bound: float, upper_bound: float):
        super().__init__()
        self.lower_bound, self.upper_bound = float(lower_bound), float(upper_bound)
        self.register_buffer("min_val", torch.tensor(lower_bound, dtype=torch.float32))
        self.register_buffer("max_val", torch.tensor(upper_bound, dtype=torch.float32))

    def forward(self, x):
        if self.training:
            min_val, max_val = x.min().detach(), x.max().detach()
            self.min_val.data, self.max_val.data = min_val, max_val
        else:
            min_val, max_val = self.min_val, self.max_val
            x = torch.maximum(torch.minimum(x, max_val), min_val)
        diff = max_val - min_val
        return (x - min_val) * (0.95 * (self.upper_bound - self.lower_bound) / diff) + \
            0.95 * self.lower_bound


class GPRegressionModel(torch.nn.Module):
    """
    DKL GPR module with the constructor of the reference (atomai/nets/gp.py:29-60):
    feature extractor -> ScaleToBounds(-1, 1) -> ConstantMean + ScaleKernel(RBFKernel(ARD)) per
    output, Gaussian likelihood.  The reference wraps the base kernel in gpytorch's KISS-GP
    (GridInterpolationKernel) and leaves every GP computation (CG, Lanczos, posterior caches) to
    gpytorch, which is neither vendored nor installed here.  This class evaluates the SAME base
    kernel densely on the native kernels (fcFeatureExtractor as wgmma 1x1 convolutions, Gram with
    the exponentiation fused in the register epilogue) and does exact-GP algebra (Cholesky) with
    torch.linalg: an exact GP instead of the SKI approximation of it, for N up to ~10^4 points.
    Hyper-parameter parametrisation follows gpytorch's defaults: softplus raw parameters,
    noise >= 1e-4, zero raw initial values; `grid_size` is accepted and ignored.
    """
    def __init__(self, X: torch.Tensor, y: torch.Tensor, likelihood=None,
                 feature_extractor: torch.nn.Module = None, embedim: int = 2,
                 grid_size: int = 50) -> None:
        super().__init__()
        batch_dim = y.size(0)
        self.train_inputs = (X,)
        self.train_targets = y
        self.feature_extractor = feature_extractor
        self.scale_to_bounds = ScaleToBounds(-1., 1.)
        self.raw_constant = torch.nn.Parameter(torch.zeros(batch_dim))
        self.raw_lengthscale = torch.nn.Parameter(torch.zeros(batch_dim, embedim))
        self.raw_outputscale = torch.nn.Parameter(torch.zeros(batch_dim))
        self.raw_noise = torch.nn.Parameter(torch.zeros(batch_dim))
        self.likelihood = likelihood
        self._cache = None

    # gpytorch-style views of the hyper-parameters
    @property
    def lengthscale(self):
        return torch.nn.functional.softplus(self.raw_lengthscale)

    @property
    def outputscale(self):
        return torch.nn.functional.softplus(self.raw_outputscale)

    @property
    def noise(self):
        return torch.nn.functional.softplus(self.raw_noise) + 1e-4

    def covar_parameters(self):
        return [self.raw_lengthscale, self.raw_outputscale]

    def mean_parameters(self):
        return [self.raw_constant]

    def likelihood_parameters(self):
        return [self.raw_noise]

    def embed(self, x: torch.Tensor) -> torch.Tensor:
        return self.scale_to_bounds(self.feature_extractor(x.to(torch.float32)))

    def neg_mll(self) -> torch.Tensor:
        """-sum_b ExactMarginalLogLikelihood_b / N (gpytorch divides the mll by the number of data
        points), the loss of GPTrainer.train_step (atomai/trainers/gptrainer.py:126-137)."""
        self._cache = None
        X, y = self.train_inputs[0], self.train_targets
        z = self.embed(X)
        n = z.shape[0]
        eye = torch.eye(n, device=z.device, dtype=y.dtype)
        total = 0.0
        for b in range(y.shape[0]):
            K = dense_rbf(z, z, self.lengthscale[b], self.outputscale[b]).to(y.dtype)
            L = torch.linalg.cholesky(K + self.noise[b].to(y.dtype) * eye)
            r = (y[b] - self.raw_constant[b].to(y.dtype))[:, None]
            alpha = torch.cholesky_solve(r, L)
            mll = -0.5 * (r * alpha).sum() - torch.log(torch.diagonal(L)).sum() \
                - 0.5 * n * 1.8378770664093453
            total = total - mll / n
        return total

    @torch.no_grad()
    def posterior(self, x_new: torch.Tensor):
        """Latent posterior mean and variance at x_new for every output: (B, n_new) each."""
        X, y = self.train_inputs[0], self.train_targets
        if self._cache is None:
            z = self.embed(X)
            eye = torch.eye(z.shape[0], device=z.device, dtype=y.dtype)
            Ls, alphas = [], []
            for b in range(y.shape[0]):
                K = dense_rbf(z, z, self.lengthscale[b], self.outputscale[b]).to(y.dtype)
                L = torch.linalg.cholesky(K + self.noise[b].to(y.dtype) * eye)
                r = (y[b] - self.raw_constant[b].to(y.dtype))[:, None]
                Ls.append(L)
                alphas.append(torch.cholesky_solve(r, L))
            self._cache = (z, Ls, alphas)
        z, Ls, alphas = self._cache
        zs = self.embed(x_new)
        means, vars_ = [], []
        for b in range(y.shape[0]):
            Ks = dense_rbf(z, zs, self.lengthscale[b], self.outputscale[b]).to(y.dtype)
            means.append((Ks.t() @ alphas[b]).squeeze(1) + self.raw_constant[b].to(y.dtype))
            v = torch.linalg.solve_triangular(Ls[b], Ks, upper=False)
            vars_.append((self.outputscale[b].to(y.dtype) - (v * v).sum(0)).clamp_min(1e-10))
        return torch.stack(means), torch.stack(vars_)


class _ExactGramFn(torch.autograd.Function):
    """K + noise I of the exact GP in float64 on the native kernels (atomai_b200_gram_f64: coordinate
    differences, float64 throughout, so the matrix is symmetric positive definite to float64
    rounding) and its hyper-parameter adjoint (atomai_b200_gram_f64_adjoint):
        dls_k = os sum_ij G_ij m_ij t_ijk^2 / ls_k,   dos = sum_ij G_ij k_ij,   dnoise = tr G
    with t_ijk = (z_ik - z_jk) / ls_k, k the unit-outputscale kernel, m = -2 dk/dr^2."""

    @staticmethod
    def forward(ctx, z, ls, os_, noise, kind):
        inv_ls = (1.0 / ls.detach().to(torch.float64)).reshape(-1).contiguous()
        n = z.shape[0]
        K = torch.empty((n, n), device=z.device, dtype=torch.float64)
        ops.gram_f64(z, inv_ls, float(os_), float(noise), _KIND[kind], K)
        ctx.save_for_backward(z, inv_ls, ls, os_, noise)
        ctx.kind = kind
        return K

    @staticmethod
    def backward(ctx, G):
        z, inv_ls, ls, os_, noise = ctx.saved_tensors
        d = z.shape[1]
        s = torch.empty(d + 2, device=z.device, dtype=torch.float64)
        ops.gram_f64_adjoint(z, inv_ls, _KIND[ctx.kind], G.contiguous(), s)
        dls = (os_.detach().to(torch.float64) * s[:d] * inv_ls).to(ls.dtype).reshape(ls.shape)
        return (None, dls, s[d].to(os_.dtype).reshape(os_.shape),
                s[d + 1].to(noise.dtype).reshape(noise.shape), None)


_KIND = {"rbf": 0, "matern": 1}


class CustomGPModel(torch.nn.Module):
    """
    Exact GP of the Reconstructor (atomai/nets/gp.py:63-128): ConstantMean + ScaleKernel(RBFKernel |
    MaternKernel(nu=2.5), ARD) on the raw inputs, Gaussian likelihood.  The reference wraps the base
    kernel in gpytorch's KISS-GP (GridInterpolationKernel); here the Gram is evaluated densely on
    the native kernels and the GP algebra is a float64 Cholesky (torch.linalg) — an exact GP in
    place of the SKI approximation of it, so `grid_points_ratio` is accepted and ignored.

    The hyper-parameters restate gpytorch's parametrisation (gpytorch is a third-party dependency
    of the reference, not vendored and not installed here, so the restatement is not checked
    against it):
      lengthscale = softplus(raw), or with `lengthscale_constraints` = (lower, upper) gpytorch's
                    Interval: lower + (upper - lower) * sigmoid(raw); raw starts at 0 either way
                    (an Interval without an initial value leaves the raw parameter alone, so the
                    lengthscale starts at the midpoint);
      outputscale = softplus(raw), noise = softplus(raw) + 1e-4, mean constant = raw; all raw
                    values start at 0.
    The raw parameters are float32 (the native Adam updates them); the training Gram, its adjoint
    and the algebra are float64 (_ExactGramFn), the predictive mean is summed in float64.
    """
    def __init__(self, train_x: torch.Tensor, train_y: torch.Tensor, likelihood=None,
                 kernel_type: str = "kissgp", base_kernel="rbf", inducing_points=None,
                 grid_points_ratio: float = 1.0, lengthscale_constraints=None, **kwargs):
        super().__init__()
        if isinstance(base_kernel, str):
            if base_kernel not in ("rbf", "matern"):
                raise ValueError("base_kernel must be either 'rbf', 'matern', or a custom "
                                 "gpytorch.kernels.Kernel object")
        else:
            raise NotImplementedError("custom base kernel objects are not supported: the native "
                                      "Gram kernels implement 'rbf' and 'matern' (nu=2.5) only")
        if kernel_type == "sparse":
            raise NotImplementedError("kernel_type='sparse' (inducing-point kernel) is not "
                                      "implemented; use kernel_type='kissgp' (exact GP)")
        if kernel_type != "kissgp":
            raise ValueError(f"Invalid kernel_type: {kernel_type}. "
                             "Supported values are 'sparse' and 'kissgp'.")
        if inducing_points is not None:
            raise NotImplementedError("inducing_points belong to the sparse kernel, which is not "
                                      "implemented")
        d = train_x.shape[-1]
        if not 1 <= d <= 4:
            raise NotImplementedError(f"the native GP mean kernel takes 1 to 4 input dimensions, "
                                      f"got {d}")
        self.kind = base_kernel
        self.train_inputs = (train_x,)
        self.train_targets = train_y.reshape(-1)
        self.raw_constant = torch.nn.Parameter(torch.zeros(()))
        self.raw_lengthscale = torch.nn.Parameter(torch.zeros(1, d))
        self.raw_outputscale = torch.nn.Parameter(torch.zeros(()))
        self.raw_noise = torch.nn.Parameter(torch.zeros(1))
        self.interval = lengthscale_constraints is not None and len(lengthscale_constraints) > 0
        lo, hi = (lengthscale_constraints if self.interval else ([0.0] * d, [0.0] * d))
        self.register_buffer("ls_lower", torch.as_tensor(lo, dtype=torch.float32).reshape(-1))
        self.register_buffer("ls_upper", torch.as_tensor(hi, dtype=torch.float32).reshape(-1))
        if self.interval and not bool((self.ls_lower < self.ls_upper).all()):
            raise ValueError("Got parameter bounds with empty intervals.")
        self.likelihood = likelihood
        self._cache = None

    @property
    def lengthscale(self) -> torch.Tensor:
        if self.interval:
            return self.ls_lower + (self.ls_upper - self.ls_lower) * torch.sigmoid(self.raw_lengthscale)
        return torch.nn.functional.softplus(self.raw_lengthscale)

    @property
    def outputscale(self) -> torch.Tensor:
        return torch.nn.functional.softplus(self.raw_outputscale)

    @property
    def noise(self) -> torch.Tensor:
        return torch.nn.functional.softplus(self.raw_noise) + 1e-4

    @property
    def constant(self) -> torch.Tensor:
        return self.raw_constant

    def covar_parameters(self):
        return [self.raw_lengthscale, self.raw_outputscale]

    def mean_parameters(self):
        return [self.raw_constant]

    def likelihood_parameters(self):
        return [self.raw_noise]

    def _inputs64(self, x: torch.Tensor) -> torch.Tensor:
        # coordinates relative to the rounded training mean: the distances are unchanged, integer
        # pixel indices stay integers (exact in fp32 for the mean kernel) and small
        return (x.to(torch.float64) - self._center).contiguous()

    def _inputs(self, x: torch.Tensor) -> torch.Tensor:
        return self._inputs64(x).to(torch.float32).contiguous()

    def _set_center(self) -> None:
        self._center = self.train_inputs[0].to(torch.float64).mean(0).round()

    def neg_mll(self) -> torch.Tensor:
        """-ExactMarginalLogLikelihood / N (gpytorch divides by the number of data points), the
        loss of GPTrainer.train_step (atomai/trainers/gptrainer.py:126-137)."""
        self._cache = None
        self._set_center()
        z = self._inputs64(self.train_inputs[0])
        n = z.shape[0]
        Kn = _ExactGramFn.apply(z, self.lengthscale.reshape(-1), self.outputscale, self.noise,
                                self.kind)
        L = torch.linalg.cholesky(Kn)
        del Kn
        r = (self.train_targets.to(torch.float64) - self.constant.to(torch.float64))[:, None]
        alpha = torch.cholesky_solve(r, L)
        mll = -0.5 * (r * alpha).sum() - torch.log(torch.diagonal(L)).sum() \
            - 0.5 * n * 1.8378770664093453
        return -mll / n

    @torch.no_grad()
    def _weights(self):
        if self._cache is None:
            self._set_center()
            z = self._inputs64(self.train_inputs[0])
            n = z.shape[0]
            ls = self.lengthscale.reshape(-1)
            K = torch.empty((n, n), device=z.device, dtype=torch.float64)
            ops.gram_f64(z, (1.0 / ls.to(torch.float64)).contiguous(), float(self.outputscale),
                         float(self.noise), _KIND[self.kind], K)
            L = torch.linalg.cholesky(K)
            del K
            r = (self.train_targets.to(torch.float64) - self.constant.to(torch.float64))[:, None]
            alpha = torch.cholesky_solve(r, L).reshape(-1).contiguous()
            self._cache = (z.to(torch.float32).contiguous(), (1.0 / ls).contiguous(), alpha)
        return self._cache

    @torch.no_grad()
    def posterior_mean(self, x_new: torch.Tensor) -> torch.Tensor:
        """Predictive mean at x_new ((n, d)) as float64, from the fused Gram-times-vector kernel
        (the n x N cross-Gram is never formed)."""
        z, inv_ls, alpha = self._weights()
        out = torch.empty(x_new.shape[0], device=z.device, dtype=torch.float64)
        ops.gram_matvec(self._inputs(x_new.to(z.device)), z, inv_ls, alpha, float(self.constant.detach()),
                        float(self.outputscale), _KIND[self.kind], out)
        return out
