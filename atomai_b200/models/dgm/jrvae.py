"""
jrVAE — rotationally (and translationally) invariant VAE with joint continuous and discrete
(Gumbel-softmax) latent variables (atomai/models/dgm/jrvae.py:23-250) on the native sm_90a path:
the joint latent kernel writes the rotation angle, the scaled shift and the decoder's latent input
in the layout the fused spatial decoder (rDecoderNet.decode) takes.
"""
from typing import List, Optional, Union

import numpy as np
import torch

from ...utils.nn import set_train_rng
from .jvae import joint_fit, joint_forward_compute_elbo
from .vae import BaseVAE


class jrVAE(BaseVAE):
    """
    Rotationally invariant VAE for joint continuous and discrete latent representations.

    Args: in_dim ((height, width[, channels])), latent_dim (continuous content latents),
    discrete_dim (sizes of the Gumbel-softmax latents), nb_classes (must stay 0), translation,
    seed, and the **kwargs of init_VAE_nets (conv_encoder, numlayers_*, numhidden_*, skip, ...).

    Example:
    >>> jrvae = jrVAE((64, 64), latent_dim=2, discrete_dim=[10], conv_encoder=True)
    >>> jrvae.fit(imstack, training_cycles=100, batch_size=100, rotation_prior=np.pi/4)
    >>> z_mean, z_sd, alphas = jrvae.encode(imstack)   # z_mean: angle, dx, dy, z1, z2
    """
    def __init__(self, in_dim: int = None, latent_dim: int = 2, discrete_dim: List[int] = [2],
                 nb_classes: int = 0, translation: bool = True, seed: int = 0,
                 **kwargs: Union[int, bool, str]) -> None:
        coord = 3 if translation else 1
        super(jrVAE, self).__init__(in_dim, latent_dim, nb_classes, coord, discrete_dim, seed=seed,
                                    **kwargs)
        set_train_rng(seed)
        self.translation = translation
        self.dx_prior = None
        self.phi_prior = None
        self.kdict_ = dict(kwargs)
        self.kdict_["num_iter"] = 0

    def forward_compute_elbo(self, x: torch.Tensor, y: Optional[torch.Tensor] = None,
                             mode: str = "train", eps: Optional[torch.Tensor] = None,
                             u: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Joint rVAE forward pass with the ELBO (jrvae.py:107-151)."""
        return joint_forward_compute_elbo(self, x, y, mode, eps, u)

    def fit(self, X_train: Union[np.ndarray, torch.Tensor],
            y_train: Optional[Union[np.ndarray, torch.Tensor]] = None,
            X_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            y_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            loss: str = "mse", verbose: str = "True", **kwargs) -> None:
        """Trains the joint rVAE (jrvae.py:153-245).  loss: 'mse' or 'ce'; kwargs
        translation_prior (0.1), rotation_prior (0.1), temperature (0.67), cont_capacity /
        disc_capacity ([max, num_iters, gamma], default [5.0, 25000, 30]), training_cycles,
        batch_size, filename; verbose "True" prints the loss after every cycle."""
        self.dx_prior = kwargs.get("translation_prior", 0.1)
        self.kdict_["phi_prior"] = kwargs.get("rotation_prior", 0.1)
        joint_fit(self, X_train, y_train, X_test, y_test, loss, verbose == "True", **kwargs)
