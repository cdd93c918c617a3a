from .dgm import VAE, BaseVAE, jrVAE, jVAE, rVAE
from .dklgp import dklGPR
from .imspec import ImSpec
from .loaders import load_model
from .segmentor import Segmentor

__all__ = ["Segmentor", "ImSpec", "VAE", "rVAE", "jVAE", "jrVAE", "BaseVAE", "dklGPR", "load_model"]
