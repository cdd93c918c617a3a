"""
rVAE — rotationally (and translationally) invariant VAE (atomai/models/dgm/rvae.py:22-219) on the
native sm_90a path: convolutional (or MLP) encoder, fused coordinate-transform + per-pixel MLP
spatial decoder, fused reconstruction reduction.  The (B, H*W, 2) coordinate tensor of the
reference (rvae.py:118,140) is never materialised.
"""
from typing import Optional, Tuple, Union

import numpy as np
import torch

from ...losses_metrics.vi_losses import rvae_loss
from ...utils.nn import set_train_rng
from .vae import BaseVAE


class rVAE(BaseVAE):
    """
    Implements rotationally and translationally invariant Variational Autoencoder (VAE) based on
    the idea of "spatial decoder" by Bepler et al. (arXiv:1909.11663).

    Args: in_dim (height, width[, channels]), latent_dim, nb_classes, translation, seed and the
    **kwargs of init_VAE_nets (conv_encoder, numlayers_encoder/decoder, numhidden_*, skip, ...).

    Example:
    >>> rvae = rVAE((64, 64), latent_dim=2, conv_encoder=True)
    >>> rvae.fit(imstack, training_cycles=100, batch_size=100)
    >>> z_mean, z_sd = rvae.encode(imstack)     # columns: angle, dx, dy, z1, z2
    """
    def __init__(self, in_dim: int = None, latent_dim: int = 2, nb_classes: int = 0,
                 translation: bool = True, seed: int = 0, **kwargs: Union[int, bool, str]) -> None:
        coord = 3 if translation else 1
        super(rVAE, self).__init__(in_dim, latent_dim, nb_classes, coord, seed=seed, **kwargs)
        set_train_rng(seed)
        self.translation = translation
        self.dx_prior = None
        self.phi_prior = None
        self.kdict_["phi_prior"] = 0.1

    def elbo_fn(self, x, x_reconstr, *args, **kwargs) -> torch.Tensor:
        return rvae_loss(self.loss, self.in_dim, x, x_reconstr, *args, **kwargs)

    def forward_compute_elbo(self, x: torch.Tensor, y: Optional[torch.Tensor] = None,
                             mode: str = "train", eps: Optional[torch.Tensor] = None
                             ) -> torch.Tensor:
        """rVAE forward pass with ELBO (rvae.py:110-147).  `eps` (optional) fixes the
        reparameterisation noise (tests)."""
        if y is not None:
            raise NotImplementedError("class-conditioned rVAE is outside the native hot path")
        grad = mode != "eval"
        with torch.set_grad_enabled(grad):
            z_mean, z_logsd = self.encoder_net(x)
            if grad:
                self.kdict_["num_iter"] += 1
            z_sd = torch.exp(z_logsd)
            z = z_mean + z_sd * eps if eps is not None else self.reparameterize(z_mean, z_sd)
            phi = z[:, 0]
            if self.translation:
                dx = z[:, 1:3] * (self.dx_prior if self.dx_prior is not None else 0.1)
                zc = z[:, 3:]
            else:
                dx, zc = None, z[:, 1:]
            x_reconstr = self.decoder_net.decode(zc, phi, dx)
            return self.elbo_fn(x, x_reconstr, z_mean, z_logsd, **self.kdict_)

    def fit(self, X_train, y_train=None, X_test=None, y_test=None, loss: str = "mse", **kwargs):
        """Trains rVAE model (rvae.py:149-215): kwargs rotation_prior, translation_prior,
        capacity, training_cycles, batch_size, filename."""
        self._check_inputs(X_train, y_train, X_test, y_test)
        self.dx_prior = kwargs.get("translation_prior", 0.1)
        self.kdict_["phi_prior"] = kwargs.get("rotation_prior", 0.1)
        for k, v in kwargs.items():
            if k in ["capacity"]:
                self.kdict_[k] = v
        self.compile_trainer((X_train, y_train), (X_test, y_test) if X_test is not None else None,
                             **{k: v for k, v in kwargs.items()
                                if k in ("training_cycles", "batch_size", "filename",
                                         "memory_alloc", "optimizer")})
        self.loss = loss
        self._fit_loop(**kwargs)
