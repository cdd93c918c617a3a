from .jrvae import jrVAE
from .jvae import jVAE
from .rvae import rVAE
from .vae import VAE, BaseVAE

__all__ = ["BaseVAE", "VAE", "rVAE", "jVAE", "jrVAE"]
