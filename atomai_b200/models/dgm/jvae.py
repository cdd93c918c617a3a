"""
jVAE — VAE with joint continuous and discrete (Gumbel-softmax) latent variables
(atomai/models/dgm/jvae.py:23-237) on the native sm_90a path.  Between the encoder heads and the
decoder, the reference's per-head softmax / log / Gumbel / tau-softmax / concat ops and the three
KL terms run as one fused kernel pair (losses_metrics/vi_losses.py: joint_latent); encoder,
decoder, reconstruction loss and the Adam step are the same kernels VAE uses.
"""
from typing import List, Optional, Union

import numpy as np
import torch

from ...losses_metrics.vi_losses import joint_elbo, joint_latent, reconstruction_loss
from ...utils.nn import set_train_rng
from .vae import BaseVAE

_TRAINER_KWARGS = ("training_cycles", "batch_size", "filename", "memory_alloc", "optimizer")


def joint_forward_compute_elbo(m: BaseVAE, x: torch.Tensor, y: Optional[torch.Tensor], mode: str,
                               eps: Optional[torch.Tensor], u: Optional[torch.Tensor]
                               ) -> torch.Tensor:
    """Training / evaluation step of jVAE and jrVAE (jvae.py:96-131, jrvae.py:107-151).  `eps`
    (B, latent_dim + coord) and `u` (B, sum(discrete_dim)) optionally fix the normal and the
    uniform noise (tests)."""
    if y is not None:
        raise NotImplementedError("class-conditioned joint VAEs are outside the native hot path")
    grad = mode != "eval"
    x = x.to(m.device)
    with torch.set_grad_enabled(grad):
        z_mean, z_logsd, logits = m.encoder_net.heads(x)
        if grad:
            m.kdict_["num_iter"] += 1
        if eps is None:
            eps = torch.randn_like(z_mean)
        dx_prior = getattr(m, "dx_prior", None)
        _, zdec, phi, dx, kl = joint_latent(
            z_mean, z_logsd, logits, m.discrete_dim, m.kdict_.get("temperature", .67), eps, u,
            coord=m.coord, phi_prior=m.kdict_.get("phi_prior", 0.1),
            dx_prior=dx_prior if dx_prior is not None else 0.1)
        if m.coord:
            x_reconstr = m.decoder_net.decode(zdec, phi, dx if m.coord == 3 else None)
        else:
            x_reconstr = m.decoder_net(zdec)
        likelihood = -reconstruction_loss(m.loss, m.in_dim, x, x_reconstr).mean()
        return joint_elbo(likelihood, kl[0], kl[1], m.discrete_dim, **m.kdict_)


def joint_fit(m: BaseVAE, X_train, y_train, X_test, y_test, loss: str, print_stats: bool,
              **kwargs) -> None:
    """fit() of jVAE / jrVAE (jvae.py:133-232, jrvae.py:153-245)."""
    if y_train is not None:
        raise NotImplementedError("class-conditioned joint VAEs are outside the native hot path")
    m._check_inputs(X_train, y_train, X_test, y_test)
    for k, v in kwargs.items():
        if k in ["cont_capacity", "disc_capacity", "temperature"]:
            m.kdict_[k] = v
    m.compile_trainer((X_train, y_train), (X_test, y_test) if X_test is not None else None,
                      **{k: v for k, v in kwargs.items() if k in _TRAINER_KWARGS})
    m.loss = loss
    if m.loss == "ce":
        m.sigmoid_out = True              # sigmoid on the decoder output at prediction time
        m.metadict["sigmoid_out"] = True
    m._fit_loop(print_stats, **kwargs)


class jVAE(BaseVAE):
    """
    VAE for joint (continuous + discrete) latent representations (atomai/models/dgm/jvae.py).

    Args: in_dim ((height, width[, channels]) or (length,)), latent_dim (continuous latents),
    discrete_dim (sizes of the Gumbel-softmax latents), nb_classes (must stay 0: class
    conditioning is not on the native path), seed, and the **kwargs of init_VAE_nets
    (conv_encoder, conv_decoder, numlayers_*, numhidden_*, skip, ...).

    Example:
    >>> jvae = jVAE((28, 28), latent_dim=2, discrete_dim=[10], numhidden_encoder=512)
    >>> jvae.fit(imstack, training_cycles=100, batch_size=100)
    >>> z_mean, z_sd, alphas = jvae.encode(imstack)
    """
    def __init__(self, in_dim: int = None, latent_dim: int = 2, discrete_dim: List[int] = [2],
                 nb_classes: int = 0, seed: int = 0, **kwargs: Union[int, bool, str]) -> None:
        super(jVAE, self).__init__(in_dim, latent_dim, nb_classes, 0, discrete_dim, seed=seed,
                                   **kwargs)
        set_train_rng(seed)
        self.kdict_ = dict(kwargs)
        self.kdict_["num_iter"] = 0

    def forward_compute_elbo(self, x: torch.Tensor, y: Optional[torch.Tensor] = None,
                             mode: str = "train", eps: Optional[torch.Tensor] = None,
                             u: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Joint VAE forward pass with the ELBO (jvae.py:96-131)."""
        return joint_forward_compute_elbo(self, x, y, mode, eps, u)

    def fit(self, X_train: Union[np.ndarray, torch.Tensor],
            y_train: Optional[Union[np.ndarray, torch.Tensor]] = None,
            X_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            y_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            loss: str = "mse", **kwargs) -> None:
        """Trains the joint VAE (jvae.py:133-232).  loss: 'mse' or 'ce'; kwargs temperature
        (0.67), cont_capacity / disc_capacity ([max, num_iters, gamma], default
        [5.0, 25000, 30]), training_cycles, batch_size, filename."""
        joint_fit(self, X_train, y_train, X_test, y_test, loss, True, **kwargs)
