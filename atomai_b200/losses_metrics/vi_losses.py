"""
ELBO terms for the VAEs with the reference's function names and maths
(atomai/losses_metrics/vi_losses.py:13-137).  The reconstruction term — the only part that touches
image-sized tensors (2*B*H*W*4 bytes) — is one fused per-sample reduction kernel that also emits
d/dx_hat for the backward pass; the KL terms act on (B, latent) tensors and stay in torch.
"""
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .. import ops


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
