"""
ImSpec — image -> spectrum / spectrum -> image model, drop-in for atomai.models.ImSpec
(atomai/models/imspec.py:18-170), trained through the native sm_90a SignalED graph.
"""
from typing import Optional, Tuple, Type, Union

import numpy as np
import torch

from ..trainers import ImSpecTrainer
from ..utils.preproc import torch_format_image, torch_format_spectra


class ImSpec(ImSpecTrainer):
    """
    Model for predicting spectra from images and vice versa.
    Args: in_dim, out_dim, latent_dim and the kwargs of init_imspec_model
    (nblayers_encoder/decoder, nbfilters_encoder/decoder, batch_norm, ...).

    Example:
    >>> model = ImSpec((64, 64), (128,), latent_dim=10)
    >>> model.fit(imgs_train, spectra_train, imgs_test, spectra_test, training_cycles=100)
    >>> prediction = model.predict(imgs_test)
    """
    def __init__(self, in_dim: Tuple[int], out_dim: Tuple[int], latent_dim: int = 2,
                 **kwargs) -> None:
        super(ImSpec, self).__init__(in_dim, out_dim, latent_dim, **kwargs)

    def fit(self, X_train, y_train, X_test=None, y_test=None, loss: str = 'mse',
            optimizer: Optional[Type[torch.optim.Optimizer]] = None, training_cycles: int = 1000,
            batch_size: int = 64, compute_accuracy: bool = False, full_epoch: bool = False,
            swa: bool = False, perturb_weights: bool = False, **kwargs):
        """Compiles a trainer and performs model training (imspec.py:63-145)."""
        self._check_upsampling()
        self.compile_trainer((X_train, y_train, X_test, y_test), loss, optimizer, training_cycles,
                             batch_size, compute_accuracy, full_epoch, swa, perturb_weights,
                             **kwargs)
        self.run()

    def predict(self, data: np.ndarray, **kwargs) -> np.ndarray:
        """Apply the (trained) model to new data (imspec.py:147-163): returns (n, *out_dim)."""
        self._check_upsampling()
        norm = kwargs.get("norm", False)
        if len(self.in_dim) == 2:
            x = torch_format_image(data, norm)
        else:
            x = torch_format_spectra(data, norm)
        num_batches = kwargs.get("num_batches", 10)
        bs = max(len(x) // num_batches, 1)
        self.net.eval()
        outs = []
        with torch.no_grad():
            for i in range(0, len(x), bs):
                outs.append(self.net(x[i:i + bs].to(self.device)).cpu())
        out = torch.cat(outs).numpy()
        return out[:, 0] if out.shape[1] == 1 else out

    def _check_upsampling(self) -> None:
        """The 1-D decoder_upsampling path starts from length // 4 and doubles twice, so it can only
        produce lengths that are multiples of 4 (the reference fails at the first loss otherwise)."""
        if self.meta_state_dict.get("decoder_upsampling") and len(self.out_dim) == 1 \
                and self.out_dim[0] % 4:
            raise ValueError(f"decoder_upsampling=True needs a spectrum length that is a multiple "
                             f"of 4, got out_dim={tuple(self.out_dim)}")
