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
    dense kernel is exposed for the covariance evaluation itself (SURVEY.md §0.6, §8a a15-a16).
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
               outputscale: float = 1.0, kind: str = "rbf") -> torch.Tensor:
    """K[i, j] = outputscale * k(||(x1_i - x2_j) / lengthscale||) with gpytorch's RBFKernel /
    MaternKernel(nu=2.5) + ScaleKernel definitions, as one fused tiled kernel (no n1 x n2 distance
    matrix in HBM, exponentiation in the epilogue).  Forward only."""
    assert x1.is_cuda and x1.dtype == torch.float32 and x1.dim() == 2 and x2.dim() == 2
    inv_ls = (1.0 / lengthscale.to(x1.device, torch.float32).reshape(-1)).contiguous()
    if inv_ls.numel() == 1:
        inv_ls = inv_ls.expand(x1.shape[1]).contiguous()
    n2 = x2.shape[0]      # row stride padded to 16 B so that the tensor-core path applies
    out = torch.empty((x1.shape[0], -(-n2 // 4) * 4), device=x1.device, dtype=torch.float32)[:, :n2]
    ops.gram(x1.contiguous(), x2.contiguous(), inv_ls, float(outputscale),
             {"rbf": 0, "matern": 1}[kind], out, engine._MATH["mode"])
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
    """K = outputscale * exp(-0.5 * ||(z1 - z2) / ls||^2) with the native Gram kernel forward and
    its adjoint built from the kernel output: with W = dK * K,
        dz1 = -(rowsum(W) * z1 - W z2) / ls^2        dz2 = -(colsum(W) * z2 - W^T z1) / ls^2
        dls = sum_ij W_ij (z1_i - z2_j)^2 / ls^3      dos = sum(dK * K) / os
    (the two n x n x d products run on the library's own GEMM kernel)."""

    @staticmethod
    def forward(ctx, z1, z2, ls, os_):
        K = dense_gram(z1, z2, ls.detach(), float(os_), "rbf")
        ctx.save_for_backward(z1, z2, ls, os_, K)
        return K

    @staticmethod
    def backward(ctx, dK):
        z1, z2, ls, os_, K = ctx.saved_tensors
        W = (dK.to(torch.float32) * K).contiguous()
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
        return dz1, dz2, dls, dos


def dense_rbf(z1, z2, lengthscale, outputscale):
    """Differentiable dense ScaleKernel(RBFKernel(ard)) Gram on the native kernels."""
    return _DenseGramFn.apply(z1, z2, lengthscale, outputscale)


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
