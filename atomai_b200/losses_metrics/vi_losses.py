"""
ELBO terms for the VAEs with the reference's function names and maths
(atomai/losses_metrics/vi_losses.py:13-251).  The reconstruction term — the only part that touches
image-sized tensors (2*B*H*W*4 bytes) — is one fused per-sample reduction kernel that also emits
d/dx_hat for the backward pass; the KL terms of VAE / rVAE act on (B, latent) tensors and stay in
torch.  For jVAE / jrVAE the whole latent block between the encoder heads and the decoder (head
softmax, both reparameterisations, the decoder input and the KL means) is one forward and one
backward kernel (`joint_latent`); only the scalar capacity terms stay in torch.
"""
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _C, ops


class _RowLossFn(torch.autograd.Function):
    """Per-sample reconstruction loss (B,) from the fused row-reduction kernel; gradient only
    w.r.t. x_hat.  kind 0: 0.5 * sum_px (x_hat - x)^2, kind 1: sum_px BCE-with-logits."""

    @staticmethod
    def forward(ctx, x, x_hat, kind):
        if not x_hat.is_cuda:
            raise RuntimeError("atomai_b200 losses run on CUDA (sm_90a) only")
        xc = x.detach().float().contiguous()
        xh = x_hat.detach().float().contiguous()
        assert xc.numel() == xh.numel(), "input and reconstruction differ in size"
        acc = torch.zeros(xc.shape[0], device=xh.device, dtype=torch.float64)
        ops.rowloss(xc, xh, kind, acc)
        ctx.save_for_backward(xc, xh)
        ctx.shape, ctx.kind = x_hat.shape, kind
        return acc.float()

    @staticmethod
    def backward(ctx, g):
        xc, xh = ctx.saved_tensors
        d = torch.empty_like(xh)
        ops.rowloss(xc, xh, ctx.kind, None, d, g.detach().float().contiguous())
        return None, d.reshape(ctx.shape), None


def reconstruction_loss(loss_type: str, in_dim: Tuple[int], x: torch.Tensor,
                        x_reconstr: torch.Tensor, logits: bool = True) -> torch.Tensor:
    """
    Reconstruction loss (mse or cross-entropy) without mean reduction, one value per sample
    (vi_losses.py:13-37), as ONE fused reduction kernel that also yields d/dx_hat.  For
    multi-channel 'ce' the reference sums over the channel axis only and leaves (B, H*W); every
    caller takes `.mean()` of the result, so the per-sample sums are divided by H*W here.
    """
    if loss_type == "mse":
        return _RowLossFn.apply(x, x_reconstr, 0)
    if loss_type == "ce":
        if not logits:
            raise NotImplementedError("'ce' reconstruction loss expects decoder logits")
        per = _RowLossFn.apply(x, x_reconstr, 1)
        if len(in_dim) == 3:
            per = per / float(int(in_dim[0]) * int(in_dim[1]))
        return per
    raise NotImplementedError("Reconstruction loss must be 'mse' or 'ce'")


def kld_normal(q_param: Tuple[torch.Tensor],
               p_param: Optional[Tuple[torch.Tensor]] = None) -> torch.Tensor:
    """KL divergence between two normal distributions, summed over the latent axis
    (vi_losses.py:40-57)."""
    mu_1, log_sd_1 = q_param
    sd_1 = torch.exp(log_sd_1)
    if p_param is None:
        kl = -log_sd_1 + 0.5 * sd_1**2 + 0.5 * mu_1**2 - 0.5
    else:
        mu_2, log_sd_2 = p_param
        sd_2 = torch.exp(log_sd_2)
        kl = (log_sd_2 - log_sd_1 + 0.5 * (sd_1**2 + (mu_1 - mu_2)**2) / sd_2**2 - 0.5)
    return torch.sum(kl, -1)


def kld_rot(phi_prior: float, phi_logsd: torch.Tensor) -> torch.Tensor:
    """KL divergence for the rotation latent variable (vi_losses.py:77-84)."""
    phi_sd = torch.exp(phi_logsd)
    return -phi_logsd + np.log(phi_prior) + phi_sd**2 / (2 * phi_prior**2) - 0.5


def infocapacity(kl_div: torch.Tensor, capacity: List[float], **kwargs) -> torch.Tensor:
    """Controlled capacity increase (vi_losses.py:224-251)."""
    num_iter = kwargs.get("num_iter", 0)
    cap_min, cap_max, cap_num_iter, cap_gamma = capacity
    cap_current = min((cap_max - cap_min) * num_iter / float(cap_num_iter) + cap_min, cap_max)
    return cap_gamma * torch.abs(cap_current - kl_div)


def vae_loss(recon_loss: str, in_dim: Tuple[int], x: torch.Tensor, x_reconstr: torch.Tensor,
             *args: torch.Tensor, **kwargs: List[float]) -> torch.Tensor:
    """ELBO of a plain VAE (vi_losses.py:87-108)."""
    if len(args) != 2:
        raise ValueError("Pass mean and SD values of encoded distribution as args")
    capacity = kwargs.get("capacity")
    likelihood = -reconstruction_loss(recon_loss, in_dim, x, x_reconstr).mean()
    kl_div = kld_normal(args).mean()
    if capacity is not None:
        kl_div = infocapacity(kl_div, capacity, num_iter=kwargs.get("num_iter", 0))
    return likelihood - kl_div


def rvae_loss(recon_loss: str, in_dim: Tuple[int], x: torch.Tensor, x_reconstr: torch.Tensor,
              *args: torch.Tensor, **kwargs: Union[List[float], float]) -> torch.Tensor:
    """ELBO of the rotationally invariant VAE (vi_losses.py:111-137): the angle's mean is dropped
    from the KL term, translations stay inside kld_normal."""
    if len(args) != 2:
        raise ValueError("Pass mean and SD values of encoded distribution as args")
    z_mean, z_logsd = args
    phi_prior = kwargs.get("phi_prior", 0.1)
    capacity = kwargs.get("capacity")
    phi_logsd = z_logsd[:, 0]
    z_mean, z_logsd = z_mean[:, 1:], z_logsd[:, 1:]
    likelihood = -reconstruction_loss(recon_loss, in_dim, x, x_reconstr).mean()
    kl_div = kld_normal([z_mean, z_logsd]).mean() + kld_rot(phi_prior, phi_logsd).mean()
    if capacity is not None:
        kl_div = infocapacity(kl_div, capacity, num_iter=kwargs.get("num_iter", 0))
    return likelihood - kl_div


def kld_discrete(alpha: torch.Tensor) -> torch.Tensor:
    """KL divergence between a Gumbel-softmax distribution with parameters `alpha` (B, D) and the
    uniform categorical distribution, batch mean, shape (1,) (vi_losses.py:60-74)."""
    eps = 1e-12
    cat_dim = alpha.size(-1)
    h1 = torch.log(alpha + eps)
    h2 = np.log(1. / cat_dim + eps)
    kld_loss = torch.mean(torch.sum(alpha * (h1 - h2), dim=1), dim=0)
    return kld_loss.view(1)


def _joint_infocapacity(kl_cont_loss: torch.Tensor, cont_capacity: List[float],
                        kl_disc_loss: torch.Tensor, disc_capacity: List[float],
                        disc_dims: List[int], num_iter: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Capacity terms of the joint VAEs (vi_losses.py:224-251): capacities [max, num_iters, gamma]
    grow linearly with the iteration count; the discrete one is also capped by sum_i log D_i."""
    cont_max, cont_num_iters, cont_gamma = cont_capacity
    cont_cap = min(cont_max * (num_iter / float(cont_num_iters)), cont_max)
    cont_capacity_loss = cont_gamma * torch.abs(kl_cont_loss - cont_cap)
    disc_max, disc_num_iters, disc_gamma = disc_capacity
    disc_theory_max = sum([float(np.log(d)) for d in disc_dims])
    disc_cap = min(disc_max * (num_iter / float(disc_num_iters)), disc_max, disc_theory_max)
    disc_capacity_loss = disc_gamma * torch.abs(disc_cap - kl_disc_loss)
    return cont_capacity_loss, disc_capacity_loss


def joint_elbo(likelihood: torch.Tensor, kl_cont: torch.Tensor, kl_disc: torch.Tensor,
               disc_dims: List[int], **kwargs: Union[List, int]) -> torch.Tensor:
    """likelihood minus both capacity terms; kwargs cont_capacity, disc_capacity (default
    [5.0, 25000, 30]) and num_iter, as the joint losses of the reference read them."""
    cont, disc = _joint_infocapacity(
        kl_cont, kwargs.get("cont_capacity", [5.0, 25000, 30]), kl_disc,
        kwargs.get("disc_capacity", [5.0, 25000, 30]), disc_dims, kwargs.get("num_iter", 0))
    return likelihood - cont - disc


def joint_vae_loss(recon_loss: str, in_dim: Tuple[int], x: torch.Tensor, x_reconstr: torch.Tensor,
                   *args: torch.Tensor, **kwargs: Union[List, int]) -> torch.Tensor:
    """Joint ELBO for continuous and discrete latent variables (vi_losses.py:140-178); args:
    z_mean, z_logsd and the list of alphas."""
    if len(args) != 3:
        raise ValueError("Pass continuous (mean, SD) and discrete (alphas) values"
                         "of encoded distributions as args")
    z_mean, z_logsd, alphas = args
    likelihood = -reconstruction_loss(recon_loss, in_dim, x, x_reconstr).mean()
    kl_cont = kld_normal([z_mean, z_logsd]).mean()
    kl_disc = torch.sum(torch.cat([kld_discrete(a) for a in alphas]))
    return joint_elbo(likelihood, kl_cont, kl_disc, [a.size(1) for a in alphas], **kwargs)


def joint_rvae_loss(recon_loss: str, in_dim: Tuple[int], x: torch.Tensor, x_reconstr: torch.Tensor,
                    *args: torch.Tensor, **kwargs: Union[List, float, int]) -> torch.Tensor:
    """Joint ELBO of the rotationally invariant joint VAE (vi_losses.py:181-221): the angle's mean
    is dropped from the continuous KL term and its log-SD enters kld_rot."""
    if len(args) != 3:
        raise ValueError("Pass continuous (mean, SD) and discrete (alphas) values"
                         "of encoded distributions as args")
    z_mean, z_logsd, alphas = args
    phi_prior = kwargs.get("phi_prior", 0.1)
    likelihood = -reconstruction_loss(recon_loss, in_dim, x, x_reconstr).mean()
    kl_cont = kld_normal([z_mean[:, 1:], z_logsd[:, 1:]]).mean() + \
        kld_rot(phi_prior, z_logsd[:, 0]).mean()
    kl_disc = torch.sum(torch.cat([kld_discrete(a) for a in alphas]))
    return joint_elbo(likelihood, kl_cont, kl_disc, [a.size(1) for a in alphas], **kwargs)


def _f32(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if t is None else t.detach().float().contiguous()


class _JointLatentFn(torch.autograd.Function):
    """The joint latent block as one autograd node over (mu, logsd, logits): forward and backward
    are one kernel launch each (atomai_b200/csrc/jlatent.cu).  The Gumbel noise is recomputed in
    the backward from the same `u` or seed."""

    @staticmethod
    def forward(ctx, desc, mode, seed, eps, u, mu, logsd, logits):
        if not logits.is_cuda:
            raise RuntimeError("atomai_b200 joint latents run on CUDA (sm_90a) only")
        ctx.set_materialize_grads(False)
        logits = _f32(logits)
        B, D = logits.shape
        dev = logits.device
        alpha = torch.empty((B, D), device=dev, dtype=torch.float32)
        mu, logsd, eps, u = _f32(mu), _f32(logsd), _f32(eps), _f32(u)
        ctx.desc, ctx.mode, ctx.seed = desc, mode, seed
        ctx.save_for_backward(mu, logsd, logits, eps, u)
        if mode == _C.JLAT_ALPHAS:
            ops.jlatent_fwd(desc, mode, None, None, logits, None, None, 0, alpha)
            return alpha
        zdec = torch.empty((B, desc.Dc - desc.coord + D), device=dev, dtype=torch.float32)
        phi = torch.empty(B, device=dev, dtype=torch.float32)
        dx = torch.empty((B, 2), device=dev, dtype=torch.float32)
        kl = torch.empty(2, device=dev, dtype=torch.float32)
        ops.jlatent_fwd(desc, mode, mu, logsd, logits, eps, u, seed, alpha, zdec, phi, dx, kl)
        return alpha, zdec, phi, dx, kl

    @staticmethod
    def backward(ctx, dalpha, *rest):
        mu, logsd, logits, eps, u = ctx.saved_tensors
        dzdec, dphi, ddx, gkl = rest if rest else (None, None, None, None)
        dlogits = torch.empty_like(logits)
        dmu = dlogsd = None
        if ctx.mode == _C.JLAT_SAMPLE:
            dmu, dlogsd = torch.empty_like(mu), torch.empty_like(logsd)
        ops.jlatent_bwd(ctx.desc, ctx.mode, mu, logsd, logits, eps, u, ctx.seed, _f32(dzdec),
                        _f32(dphi), _f32(ddx), _f32(dalpha), _f32(gkl), dmu, dlogsd, dlogits)
        return None, None, None, None, None, dmu, dlogsd, dlogits


def _check_shapes(logits, discrete_dim, mu=None, logsd=None, eps=None, u=None) -> None:
    if logits.dim() != 2 or logits.shape[1] != sum(int(d) for d in discrete_dim):
        raise ValueError(f"logits of shape {tuple(logits.shape)} for discrete heads {list(discrete_dim)}")
    if mu is not None:
        if mu.dim() != 2 or mu.shape[0] != logits.shape[0] or any(
                t.shape != mu.shape for t in (logsd, eps)):
            raise ValueError("mu, logsd and eps must be (B, Dc) matrices with the rows of logits")
        if u is not None and u.shape != logits.shape:
            raise ValueError("u must have the shape of logits")


def joint_alphas(logits: torch.Tensor, discrete_dim: List[int]) -> torch.Tensor:
    """Per-head softmax of the concatenated discrete-head logits (B, sum D) -> alphas (B, sum D)
    (the F.softmax(fc13[i](x), dim=1) of atomai/nets/ed.py:406-409, 463-466)."""
    _check_shapes(logits, discrete_dim)
    desc = ops.jlat_desc(logits.shape[0], 0, 0, discrete_dim, 1.0)
    return _JointLatentFn.apply(desc, _C.JLAT_ALPHAS, 0, None, None, None, None, logits)


def joint_latent(mu: torch.Tensor, logsd: torch.Tensor, logits: torch.Tensor,
                 discrete_dim: List[int], tau: float, eps: torch.Tensor,
                 u: Optional[torch.Tensor] = None, seed: Optional[int] = None, coord: int = 0,
                 phi_prior: float = 0.1, dx_prior: float = 0.1):
    """The sampling step of jVAE / jrVAE between the encoder heads and the decoder, fused.

    mu, logsd: (B, Dc) continuous encoder outputs (after the optional softplus); logits: (B, sum D)
    the discrete heads' logits; eps: (B, Dc) normal noise; u: (B, sum D) uniform noise, or None to
    draw the Gumbel noise from the counter-hash generator with `seed`.  coord: 0 (jVAE), 1 or 3
    (jrVAE without / with translation).  Returns (alpha, zdec, phi, dx, kl): alpha (B, sum D);
    zdec = [z[:, coord:], z_disc] the decoder input; phi = z[:, 0] and dx = z[:, 1:3] * dx_prior
    (only meaningful for coord 1 / 3); kl = [continuous KL mean (+ rotation KL mean), discrete KL
    summed over heads], all differentiable.  Limits: Dc <= 32, sum D <= 64 (ValueError beyond)."""
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if u is None else 0
    _check_shapes(logits, discrete_dim, mu, logsd, eps, u)
    desc = ops.jlat_desc(mu.shape[0], mu.shape[1], coord, discrete_dim, tau, phi_prior, dx_prior)
    return _JointLatentFn.apply(desc, _C.JLAT_SAMPLE, seed, eps, u, mu, logsd, logits)
