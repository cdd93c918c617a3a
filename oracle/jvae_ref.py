"""
TEST INFRASTRUCTURE — CPU restatement (plain torch functional ops, any float dtype) of the
reference's jVAE / jrVAE step: joint encoders, Gumbel-softmax reparameterisation, decoders, the
joint ELBO with its capacity terms.  state_dict-first like oracle/vae_ref.py.  Only tests and tools
may import it.  Parity status: PINNED by tests/test_jvae.py against goldens produced by the
unmodified reference (tests/golden/make_golden_jvae.py); the float64 form is the yardstick of the
fused joint-latent kernels in tests/test_jvae_gpu.py.
"""
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from .nets_ref import conv_block
from .vae_ref import conv_decoder, fc_decoder, imcoordgrid

SD = Dict[str, torch.Tensor]
EPS = 1e-12


def joint_encoder(x, sd: SD, conv: bool, nheads: int, num_layers=2):
    """jconvEncoderNet / jfcEncoderNet.forward (atomai/nets/ed.py:398-407, 455-468) without the
    head softmax: (z_mean, z_logsd, [head logits])."""
    if conv:
        h = x.unsqueeze(1) if x.ndim in (2, 3) else x.permute(0, -1, 1, 2)
        h = conv_block(h, sd, "conv", num_layers, False, 0.1)
    else:
        h = x.reshape(x.shape[0], -1)
        for i in range(num_layers):
            h = torch.tanh(F.linear(h, sd[f"dense.{2*i}.weight"], sd[f"dense.{2*i}.bias"]))
    h = h.reshape(h.shape[0], -1)
    lin = [F.linear(h, sd[f"{n}.weight"], sd[f"{n}.bias"])
           for n in ["fc11", "fc12"] + [f"fc13.{i}" for i in range(nheads)]]
    return lin[0], lin[1], lin[2:]


def joint_latent(mu, logsd, logits, heads: List[int], tau: float, eps, u, coord: int = 0,
                 phi_prior: float = 0.1, dx_prior: float = 0.1):
    """The block between the encoder heads and the decoder (jvae.py:110-121, jrvae.py:126-145,
    vitrainer.py:223-248, vi_losses.py:40-84,140-221): returns alpha, zdec = [z[:, coord:], zd],
    phi, dx, kl_cont, kl_disc."""
    offs = np.cumsum([0] + list(heads))
    alphas = [F.softmax(logits[:, offs[h]:offs[h + 1]], dim=1) for h in range(len(heads))]
    z = mu + torch.exp(logsd) * eps
    zd = []
    for h, a in enumerate(alphas):
        g = -torch.log(-torch.log(u[:, offs[h]:offs[h + 1]] + EPS) + EPS)
        zd.append(F.softmax((torch.log(a + EPS) + g) / tau, dim=1))
    zdec = torch.cat([z[:, coord:]] + zd, 1)
    phi = z[:, 0] if coord else None
    dx = z[:, 1:3] * dx_prior if coord == 3 else None
    if coord:
        kl_cont = kld_normal(mu[:, 1:], logsd[:, 1:]).mean() + kld_rot(phi_prior, logsd[:, 0]).mean()
    else:
        kl_cont = kld_normal(mu, logsd).mean()
    kl_disc = sum(kld_discrete(a) for a in alphas)
    return torch.cat(alphas, 1), zdec, phi, dx, kl_cont, kl_disc


def kld_normal(mu, log_sd):
    sd = torch.exp(log_sd)
    return torch.sum(-log_sd + 0.5 * sd**2 + 0.5 * mu**2 - 0.5, -1)


def kld_rot(phi_prior, phi_logsd):
    return -phi_logsd + np.log(phi_prior) + torch.exp(phi_logsd)**2 / (2 * phi_prior**2) - 0.5


def kld_discrete(alpha):
    h2 = np.log(1. / alpha.shape[1] + EPS)
    return torch.mean(torch.sum(alpha * (torch.log(alpha + EPS) - h2), dim=1), dim=0)


def capacity_terms(kl_cont, kl_disc, heads, num_iter, cont_capacity=(5.0, 25000, 30),
                   disc_capacity=(5.0, 25000, 30)):
    """infocapacity with a discrete channel (vi_losses.py:224-251)."""
    cmax, cn, cg = cont_capacity
    ccap = min(cmax * num_iter / float(cn), cmax)
    dmax, dn, dg = disc_capacity
    dcap = min(dmax * num_iter / float(dn), dmax, sum(float(np.log(d)) for d in heads))
    return cg * torch.abs(kl_cont - ccap), dg * torch.abs(dcap - kl_disc)


def r_decoder(z, phi, dx, sd: SD, hw, num_layers=2, skip=False):
    """transform_coordinates + rDecoderNet.forward (atomai/utils/coords.py:57-83,
    atomai/nets/ed.py:626-642, 672-687), c = 1."""
    b = z.shape[0]
    grid = imcoordgrid(hw).to(z.dtype).expand(b, -1, -1)
    c, s = torch.cos(phi), torch.sin(phi)
    rot = torch.stack([torch.stack([c, s], 1), torch.stack([-s, c], 1)], 1)
    coord = torch.bmm(grid, rot)
    if dx is not None:
        coord = coord + dx.unsqueeze(1)
    h = F.linear(coord.reshape(-1, 2), sd["coord_latent.fc_coord.weight"],
                 sd["coord_latent.fc_coord.bias"]).reshape(b, hw[0] * hw[1], -1)
    h = h + F.linear(z, sd["coord_latent.fc_latent.weight"]).unsqueeze(1)
    if not skip:
        h = torch.tanh(h)
    h = h.reshape(b * hw[0] * hw[1], -1)
    res = h
    for i in range(num_layers):
        h = torch.tanh(F.linear(h, sd[f"fc_decoder.{2*i}.weight"], sd[f"fc_decoder.{2*i}.bias"]))
        if skip:
            h = h + res
    return F.linear(h, sd["out.weight"], sd["out.bias"]).reshape(b, *hw)


def joint_forward(x, eps, u, enc: SD, dec: SD, hw, case: dict, hidden=128,
                  num_iter: Optional[int] = None):
    """jVAE / jrVAE.forward_compute_elbo (mse) with injected noise; case: a jvae_cases entry.
    Returns elbo, z_mean, z_logsd, alphas, z_disc, x_reconstr."""
    heads = case["discrete"]
    mu, ls, logits = joint_encoder(x, enc, case["conv"], len(heads))
    coord = 0 if case["kind"] == "jvae" else (3 if case["translation"] else 1)
    alpha, zdec, phi, dx, kl_cont, kl_disc = joint_latent(
        mu, ls, torch.cat(logits, 1), heads, case["tau"], eps, u, coord,
        case.get("phi_prior", 0.1), case.get("dx_prior", 0.1))
    if coord:
        x_rec = r_decoder(zdec, phi, dx, dec, hw, skip=case.get("skip", False))
    elif case["conv"]:
        x_rec = conv_decoder(zdec, dec, hw, hidden)
    else:
        x_rec = fc_decoder(zdec, dec, hw)
    b = x.shape[0]
    rec = 0.5 * torch.sum((x_rec.reshape(b, -1) - x.reshape(b, -1))**2, 1)
    n = case["num_iter"] + 1 if num_iter is None else num_iter
    c_loss, d_loss = capacity_terms(kl_cont, kl_disc, heads, n)
    elbo = -rec.mean() - c_loss - d_loss
    return elbo, mu, ls, alpha, zdec[:, zdec.shape[1] - sum(heads):], x_rec
