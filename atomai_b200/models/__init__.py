from .denoiser import DenoisingAutoencoder, denoise_images
from .dgm import VAE, BaseVAE, jrVAE, jVAE, rVAE
from .dklgp import Reconstructor, dklGPR
from .imspec import ImSpec
from .loaders import load_model
from .regcls import Classifier, Regressor
from .segmentor import Segmentor

__all__ = ["Segmentor", "ImSpec", "VAE", "rVAE", "jVAE", "jrVAE", "BaseVAE", "dklGPR",
           "DenoisingAutoencoder", "denoise_images", "Regressor", "Classifier", "load_model",
           "Reconstructor"]
