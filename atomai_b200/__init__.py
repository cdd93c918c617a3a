"""
atomai_b200 — H100-native (sm_90a) implementation of AtomAI's data-parallel hot path
(pycroscopy/atomai v0.8.1): Segmentor / Unet convolutional forward+backward, (r)VAE encoder /
decoder / ELBO, ImSpec, and the DKL deep-kernel Gram matrix, behind AtomAI's own Python API.

All arithmetic runs in libatomai_b200.so (hand-written CUDA: wgmma tensor-core implicit-GEMM
convolutions + HBM-bound fused kernels); there is no CPU or eager-PyTorch fallback.
"""
from .__version__ import version as __version__
from .engine import get_math, set_fusion, set_math
from . import losses_metrics, models, nets, predictors, trainers, transforms, utils

__all__ = ["nets", "losses_metrics", "trainers", "predictors", "models", "utils", "transforms",
           "set_math", "set_fusion",
           "get_math", "__version__"]
