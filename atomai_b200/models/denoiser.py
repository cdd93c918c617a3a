"""
DenoisingAutoencoder — noisy -> clean image model (train + predict), drop-in for
atomai.models.DenoisingAutoencoder (atomai/models/denoiser.py:20-270).  Training runs the
BaseTrainer loop (native forward / backward, fused MSE loss and Adam, data parallelism under
torchrun); the network is nets.DenoisingAutoencoderNet.
"""
from typing import Optional, Tuple, Type, Union

import numpy as np
import torch

from ..nets import DenoisingAutoencoderNet
from ..predictors import BasePredictor
from ..trainers import BaseTrainer
from ..utils.nn import set_train_rng
from ..utils.preproc import preprocess_denoiser_data


class DenoisingAutoencoder(BaseTrainer):
    """
    Denoising autoencoder model for image cleaning and noise reduction

    Args:
        encoder_filters: filters of the encoder blocks (Default: [8, 16, 32, 64])
        decoder_filters: filters of the decoder blocks (Default: [64, 32, 16, 8])
        encoder_layers: convolutional layers per encoder block (Default: [1, 2, 2, 2])
        decoder_layers: convolutional layers per decoder block (Default: [2, 2, 2, 1])
        use_batch_norm: batch normalization after every convolution (Default: False)
        upsampling_mode: 'nearest' or 'bilinear' (Default: 'nearest')
        **seed: random seed (Default: 1)

    Input height and width must be divisible by 2**(len(encoder_filters) - 1).

    Example:
        >>> model = DenoisingAutoencoder()
        >>> model.fit(noisy_images, clean_images, noisy_test, clean_test,
        >>>           training_cycles=500, swa=True)
        >>> cleaned = model.predict(new_noisy_images)
    """
    def __init__(self,
                 encoder_filters: list = [8, 16, 32, 64],
                 decoder_filters: list = [64, 32, 16, 8],
                 encoder_layers: list = [1, 2, 2, 2],
                 decoder_layers: list = [2, 2, 2, 1],
                 use_batch_norm: bool = False,
                 upsampling_mode: str = 'nearest',
                 **kwargs) -> None:
        super(DenoisingAutoencoder, self).__init__()
        set_train_rng(kwargs.get("seed", 1))
        self.encoder_filters = encoder_filters
        self.decoder_filters = decoder_filters
        self.encoder_layers = encoder_layers
        self.decoder_layers = decoder_layers
        self.use_batch_norm = use_batch_norm
        self.upsampling_mode = upsampling_mode
        self.net = self._build_autoencoder()
        self.net.to(self.device)
        self.meta_state_dict = {
            "model_type": "denoising_autoencoder",
            "encoder_filters": encoder_filters,
            "decoder_filters": decoder_filters,
            "encoder_layers": encoder_layers,
            "decoder_layers": decoder_layers,
            "use_batch_norm": use_batch_norm,
            "upsampling_mode": upsampling_mode,
            "weights": self.net.state_dict()
        }

    def _build_autoencoder(self) -> DenoisingAutoencoderNet:
        return DenoisingAutoencoderNet(self.encoder_filters, self.decoder_filters,
                                       self.encoder_layers, self.decoder_layers,
                                       self.use_batch_norm, self.upsampling_mode)

    def fit(self,
            X_train: Union[np.ndarray, torch.Tensor],
            y_train: Union[np.ndarray, torch.Tensor],
            X_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            y_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            loss: str = 'mse',
            optimizer: Optional[Type[torch.optim.Optimizer]] = None,
            training_cycles: int = 500,
            batch_size: int = 32,
            compute_accuracy: bool = False,
            full_epoch: bool = False,
            swa: bool = True,
            perturb_weights: bool = False,
            **kwargs):
        """
        Trains the denoising autoencoder on noisy (X) / clean (y) image pairs — arguments and
        kwargs (test_size, seed when no test set is given; lr_scheduler, batch_seed, print_loss,
        filename, memory_alloc, ...) as in atomai/models/denoiser.py:132-186.  The model has no
        accuracy metric: compute_accuracy=True raises NotImplementedError at the first step, as
        in the reference.  perturb_weights is refused with batch normalization.
        """
        if X_test is None or y_test is None:
            from sklearn.model_selection import train_test_split
            X_train, X_test, y_train, y_test = train_test_split(
                X_train, y_train, test_size=kwargs.get("test_size", .15),
                shuffle=True, random_state=kwargs.get("seed", 1))
        X_train, y_train, X_test, y_test = preprocess_denoiser_data(
            X_train, y_train, X_test, y_test)
        if perturb_weights and self.use_batch_norm:
            raise AssertionError("To use time-dependent weights perturbation, " +
                                 "turn off the batch normalization layes")
        self.compile_trainer(
            (X_train, y_train, X_test, y_test),
            loss=loss, optimizer=optimizer, training_cycles=training_cycles,
            batch_size=batch_size, compute_accuracy=compute_accuracy,
            full_epoch=full_epoch, swa=swa, perturb_weights=perturb_weights,
            **kwargs)
        self.run()
        self.meta_state_dict["weights"] = self.net.state_dict()

    def predict(self, data: Union[np.ndarray, torch.Tensor], **kwargs) -> np.ndarray:
        """
        Denoises images: numpy (h, w), (n, h, w) or (n, 1, h, w), or a (n, 1, h, w) tensor
        (**num_batches, default 1).  Returns the squeezed numpy array of the network output.
        """
        use_gpu = self.device == 'cuda'
        predictor = BasePredictor(self.net, use_gpu, **kwargs)
        if isinstance(data, np.ndarray):
            if data.ndim == 2:
                data = data[None, None, ...]
            elif data.ndim == 3:
                data = data[:, None, ...]
        prediction = predictor.predict(data, **kwargs)
        return prediction.detach().cpu().numpy().squeeze()

    def load_weights(self, filepath: str) -> None:
        """Loads a state_dict, or the 'weights' of a saved meta-state dictionary."""
        weight_dict = torch.load(filepath, map_location=self.device)
        if "weights" in weight_dict:
            self.net.load_state_dict(weight_dict["weights"])
        else:
            self.net.load_state_dict(weight_dict)


def init_denoising_autoencoder(**kwargs) -> Tuple[DenoisingAutoencoderNet, dict]:
    """Returns (net, meta_state_dict) of a DenoisingAutoencoder(**kwargs)."""
    model = DenoisingAutoencoder(**kwargs)
    return model.net, model.meta_state_dict


def denoise_images(noisy_images: np.ndarray,
                   clean_images: np.ndarray,
                   test_noisy: Optional[np.ndarray] = None,
                   test_clean: Optional[np.ndarray] = None,
                   training_cycles: int = 500,
                   **kwargs) -> Tuple[DenoisingAutoencoder, Optional[np.ndarray]]:
    """
    Trains a DenoisingAutoencoder(**kwargs) with fit(..., **kwargs) and returns
    (model, denoised test_noisy or None) — atomai/models/denoiser.py:238-270.
    """
    model = DenoisingAutoencoder(**kwargs)
    model.fit(noisy_images, clean_images, test_noisy, test_clean,
              training_cycles=training_cycles, **kwargs)
    predictions = None
    if test_noisy is not None:
        predictions = model.predict(test_noisy)
    return model, predictions
