from .dklgpr import dklGPR
from .gpr import Reconstructor

__all__ = ["dklGPR", "Reconstructor"]
