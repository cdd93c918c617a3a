"""
Reconstructor — GP reconstruction of sparsely sampled images, drop-in for
atomai.models.Reconstructor (atomai/models/dklgp/gpr.py:11-114): fit, predict, reconstruct with the
reference's argument conventions.  The GP is exact (atomai_b200.nets.gp.CustomGPModel) where the
reference runs gpytorch's KISS-GP; the predictive mean over every pixel runs on the fused
Gram-times-vector kernel, so the (pixels x measured pixels) cross-Gram is never formed.
"""
from typing import List, Optional, Tuple

import numpy as np
import torch

from ...trainers.gptrainer import GPTrainer
from ...utils.coords import get_lengthscale_constraints
from ...utils.preproc import create_batches, prepare_gp_input


class Reconstructor(GPTrainer):
    """
    Sparse image reconstructor: a Gaussian process fitted to the measured pixels of a scan,
    predicting every pixel.

    Keyword Args:
        device: 'cuda:0' by default (the native kernels have no CPU path)
        precision: 'single' (torch.float32, default) or 'double' (torch.float64) for the data and
            the predictions; the GP algebra is float64 either way
        seed: seed for reproducibility

    Examples:

        >>> rec = Reconstructor()
        >>> image = rec.reconstruct(sparse_image, training_cycles=100)
    """
    def __init__(self, **kwargs) -> None:
        super(Reconstructor, self).__init__(**kwargs)

    def fit(self, X, y, training_cycles: int, **kwargs) -> None:
        """
        Trains the GP on inputs X ((N, num_features), e.g. pixel indices) and targets y ((N,)).

        Keyword Args:
            grid_points_ratio: accepted for compatibility and ignored (the GP is exact)
            lr: learning rate of Adam (default 0.1)
            kernel_type: 'kissgp' (default; runs the exact GP); 'sparse' is not implemented
            base_kernel: 'rbf' (default) or 'matern' (nu = 2.5)
            lengthscale_constraints: optional ([lower...], [upper...]) per input dimension
            print_loss: print the loss every n-th training cycle
        """
        _ = self.run(X, y, training_cycles, **kwargs)

    def predict(self, X_new, **kwargs) -> torch.Tensor:
        """
        Predictive mean at X_new ((n, num_features)) as a tensor of the trainer's dtype.

        Keyword Args:
            batch_size: number of points per call of the mean kernel (default: all); the result does
                not depend on it
            device: device the inputs are moved to (default: the trainer's)
        """
        batch_size = kwargs.get("batch_size", len(X_new))
        device = kwargs.get("device")
        self.gp_model.eval()
        reconstruction = []
        for x in create_batches(X_new, batch_size):
            x = self._set_data(x, device)
            reconstruction.append(self.gp_model.posterior_mean(x).to(self.dtype))
        return torch.cat(reconstruction)

    def reconstruct(self, sparse_image: np.ndarray, training_cycles: int = 100,
                    lengthscale_constraints: Optional[Tuple[List[float]]] = None,
                    grid_points_ratio: float = 1.0, **kwargs) -> np.ndarray:
        """
        Trains on the non-zero pixels of `sparse_image` (unmeasured pixels must be zero) and
        returns the predicted image (same shape).  Without `lengthscale_constraints` the
        lengthscale is bounded to [1, max index // 2 + 1] per dimension.  Keyword arguments go
        to fit and predict.
        """
        X_train, y_train, X_full = prepare_gp_input(sparse_image)
        if not lengthscale_constraints:
            lengthscale_constraints = get_lengthscale_constraints(X_full)
        print("Model training ...\n")
        self.fit(X_train, y_train, training_cycles,
                 lengthscale_constraints=lengthscale_constraints,
                 grid_points_ratio=grid_points_ratio, **kwargs)
        print('\n\rPerforming reconstruction... ', end="")
        reconstruction = self.predict(X_full, **kwargs)
        print("Done")
        return reconstruction.view(sparse_image.shape).cpu().numpy()
