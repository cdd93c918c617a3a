"""
Trainers for deep-kernel-learning GP regression with the reference's public surface
(atomai/trainers/gptrainer.py:18-57, 126-349): GPTrainer data handling + train_step, dklGPTrainer
compile_trainer / compile_multi_model_trainer / run / save_weights.  The feature extractor and the
kernel Gram run on the native sm_90a kernels; the GP algebra is the dense exact GP of
atomai_b200.nets.gp.GPRegressionModel (gpytorch, which the reference delegates it to, is not
available in this image).
"""
from copy import deepcopy as dc
from typing import Optional, Tuple, Type, Union

import numpy as np
import torch

from ..nets.gp import CustomGPModel, GPRegressionModel, fcFeatureExtractor
from ..optim import FusedAdam


def set_seed_and_precision(seed: int = 42, precision: str = "double", **kwargs) -> None:
    """Seeds numpy / torch (atomai/utils/nn.py:149-166).  The reference also switches torch's
    GLOBAL default tensor type here; that process-wide side effect is deliberately not reproduced
    (dtype is carried by the trainer instead)."""
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


# float64 N x N matrices counted for an exact-GP training step: the measured peak is 6.0 (the
# Cholesky factor - K + noise is freed once factored - and the temporaries of the cholesky_solve and
# Cholesky backward passes up to the gradient of K + noise, which the adjoint kernel reads in
# place) plus O(N) vectors; one more matrix of headroom for the allocator's rounding
# (tests/test_reconstructor_gpu.py measures the peak against this count)
_EXACT_GP_NXN = 7


def check_exact_gp_memory(n: int, device) -> None:
    """Fails before anything is allocated when the float64 N x N algebra of an exact GP on n
    points cannot fit in the free memory of `device`."""
    need = _EXACT_GP_NXN * 8 * n * n
    free, _ = torch.cuda.mem_get_info(torch.device(device))
    if need > free:
        raise MemoryError(
            f"exact GP on N = {n} points needs about {need / 2**30:.1f} GiB for its float64 "
            f"N x N Cholesky algebra, {free / 2**30:.1f} GiB of device memory are free; "
            "measure fewer points (a sparser scan or a crop)")


class GPTrainer:
    def __init__(self, **kwargs: Union[str, int]) -> None:
        precision = kwargs.get("precision", "single")
        set_seed_and_precision(precision=precision)
        self.device = kwargs.get("device", 'cuda:0' if torch.cuda.is_available() else 'cpu')
        self.dtype = torch.float32 if precision == "single" else torch.float64
        self.gp_model = None
        self.likelihood = None
        self.compiled = False
        self.train_loss = []

    def _set_data(self, x, device: str = None) -> torch.Tensor:
        device_ = device if device else self.device
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(x).to(self.dtype).to(device_)
        elif isinstance(x, torch.Tensor):
            x = x.to(self.dtype).to(device_)
        else:
            raise TypeError("Pass data as ndarray or torch tensor object")
        return x

    def set_data(self, x, y=None, device: str = None) -> Tuple[torch.Tensor]:
        """Casts data to the trainer's dtype / device; 1-D targets become (1, N)."""
        x = self._set_data(x, device)
        if y is not None:
            y = y[None] if y.ndim == 1 else y
            y = self._set_data(y, device)
        return x, y

    def compile_trainer(self, X, y, training_cycles: int = 1, **kwargs) -> None:
        """Exact GP on the raw inputs (atomai/trainers/gptrainer.py:59-93): CustomGPModel with the
        kwargs kernel_type, base_kernel, inducing_points, grid_points_ratio (ignored: the GP is
        exact), lengthscale_constraints; Adam over every hyper-parameter with kwargs lr (0.1)."""
        X, y = self.set_data(X, y)
        self.gp_model = CustomGPModel(X, y, None, **kwargs)
        if not str(self.device).startswith("cuda"):
            raise RuntimeError("atomai_b200 runs on CUDA (H100, sm_90a) only: the native GP "
                               "kernels have no CPU fallback")
        check_exact_gp_memory(X.shape[0], self.device)
        self.gp_model.to(self.device)
        self.gp_model.train()
        list_of_params = [{'params': self.gp_model.covar_parameters()},
                          {'params': self.gp_model.mean_parameters()},
                          {'params': self.gp_model.likelihood_parameters()}]
        self.optimizer = FusedAdam(list_of_params, lr=kwargs.get("lr", 0.1))
        self.training_cycles = training_cycles
        self.compiled = True

    def run(self, X=None, y=None, training_cycles: int = 1, **kwargs):
        """Initializes (if needed) and trains the GP (atomai/trainers/gptrainer.py:95-124)."""
        if not self.compiled:
            self.compile_trainer(X, y, training_cycles, **kwargs)
        for e in range(self.training_cycles):
            self.train_step()
            if any([e == 0, (e + 1) % kwargs.get("print_loss", 10) == 0,
                    e == self.training_cycles - 1]):
                self.print_statistics(e)
        return self.gp_model

    def train_step(self) -> None:
        """Full-batch step on -mll (atomai/trainers/gptrainer.py:126-137)."""
        self.optimizer.zero_grad()
        models = self.gp_model.models if hasattr(self.gp_model, "models") else [self.gp_model]
        loss = sum(m.neg_mll() for m in models)
        loss.backward()
        self.optimizer.step()
        self.train_loss.append(loss.item())

    def print_statistics(self, e):
        print('Epoch {}/{} ...'.format(e+1, self.training_cycles),
              'Training loss: {}'.format(np.around(self.train_loss[-1], 4)))


class IndependentModelList(torch.nn.Module):
    """One independent GP (own feature extractor) per output — the role of
    gpytorch.models.IndependentModelList in atomai/trainers/gptrainer.py:223-226."""
    def __init__(self, *models):
        super().__init__()
        self.models = torch.nn.ModuleList(models)

    @property
    def train_targets(self):
        return [m.train_targets for m in self.models]

    @property
    def train_inputs(self):
        return [m.train_inputs for m in self.models]


class dklGPTrainer(GPTrainer):
    """
    Deep kernel learning (DKL)-based Gaussian process regression (GPR)

    Args: indim, embedim, shared_embedding_space and the kwargs device, precision ('single' |
    'double': the feature extractor always computes in fp32 on the tensor cores; 'double' runs the
    GP algebra in float64), seed — atomai/trainers/gptrainer.py:144-179.
    """
    def __init__(self, indim: int, embedim: int = 2, shared_embedding_space: bool = True,
                 **kwargs: Union[str, int]) -> None:
        super(dklGPTrainer, self).__init__(**kwargs)
        set_seed_and_precision(**kwargs)
        self.dimdict = {"input_dim": indim, "embedim": embedim}
        self.device = kwargs.get("device", 'cuda:0' if torch.cuda.is_available() else 'cpu')
        precision = kwargs.get("precision", "double")
        self.dtype = torch.float32 if precision == "single" else torch.float64
        self.correlated_output = shared_embedding_space
        self.ensemble = False

    def _require_cuda(self):
        if not str(self.device).startswith("cuda"):
            raise RuntimeError("atomai_b200 runs on CUDA (H100, sm_90a) only: the native deep-"
                               "kernel path has no CPU fallback")

    def _optimizer(self, param_groups, lr):
        return FusedAdam(param_groups, lr=lr)

    def compile_multi_model_trainer(self, X, y, training_cycles: int = 1, **kwargs) -> None:
        """One feature extractor + GP per output (or per ensemble member):
        atomai/trainers/gptrainer.py:181-244."""
        if self.correlated_output:
            raise NotImplementedError(
                "To compile a DKL-GP trainer for correlated outputs " +
                "use compile_trainer(*args, **kwargs)")
        self._require_cuda()
        X, y = self.set_data(X, y)
        if y.shape[0] < 2:
            raise ValueError("The training targets must be vector-valued (d >1)")
        input_dim, embedim = self.dimdict["input_dim"], self.dimdict["embedim"]
        feature_net = kwargs.get("feature_extractor", fcFeatureExtractor)
        freeze_weights = kwargs.get("freeze_weights", False)
        if not self.ensemble:
            feature_extractor = feature_net(input_dim, embedim)
            if freeze_weights:
                for p in feature_extractor.parameters():
                    p.requires_grad = False
        list_of_models = []
        for i in range(y.shape[0]):
            if self.ensemble:  # different initialization for each model
                feature_extractor = feature_net(input_dim, embedim)
                if freeze_weights:
                    for p in feature_extractor.parameters():
                        p.requires_grad = False
            model_i = GPRegressionModel(X, y[i:i+1], None, feature_extractor, embedim,
                                        kwargs.get("grid_size", 50))
            list_of_models.append(dc(model_i))
        self.gp_model = IndependentModelList(*list_of_models)
        self.likelihood = None
        self.gp_model.to(self.device)
        list_of_parameters = []
        for m in self.gp_model.models:
            list_of_parameters += m.covar_parameters() + m.mean_parameters() + \
                m.likelihood_parameters()
            if not freeze_weights:
                list_of_parameters += list(m.feature_extractor.parameters())
        self.optimizer = self._optimizer(list_of_parameters, 0.01)
        self.training_cycles = training_cycles
        self.compiled = True

    def compile_trainer(self, X, y, training_cycles: int = 1, **kwargs) -> None:
        """Shared embedding space: one feature extractor feeding one GP per output
        (atomai/trainers/gptrainer.py:246-305); kwargs feature_extractor, grid_size (ignored: the
        kernel is evaluated densely), freeze_weights, lr."""
        if not self.correlated_output:
            raise NotImplementedError(
                "To compile a DKL-GP trainer for independent outputs " +
                "use compile_multi_model_trainer(*args, **kwargs)")
        self._require_cuda()
        X, y = self.set_data(X, y)
        input_dim, embedim = self.dimdict["input_dim"], self.dimdict["embedim"]
        feature_net = kwargs.get("feature_extractor", fcFeatureExtractor)
        feature_extractor = feature_net(input_dim, embedim)
        freeze_weights = kwargs.get("freeze_weights", False)
        if freeze_weights:
            for p in feature_extractor.parameters():
                p.requires_grad = False
        self.gp_model = GPRegressionModel(X, y, None, feature_extractor, embedim,
                                          kwargs.get("grid_size", 50))
        self.likelihood = None
        self.gp_model.to(self.device)
        self.gp_model.train()
        list_of_params = [{'params': self.gp_model.covar_parameters()},
                          {'params': self.gp_model.mean_parameters()},
                          {'params': self.gp_model.likelihood_parameters()}]
        if not freeze_weights:
            list_of_params.append({'params': list(self.gp_model.feature_extractor.parameters())})
        self.optimizer = self._optimizer(list_of_params, kwargs.get("lr", 0.01))
        self.training_cycles = training_cycles
        self.compiled = True

    def run(self, X=None, y=None, training_cycles: int = 1, **kwargs):
        """Initializes (if needed) and trains a deep kernel GP model
        (atomai/trainers/gptrainer.py:307-341)."""
        if not self.compiled:
            if self.correlated_output:
                self.compile_trainer(X, y, training_cycles, **kwargs)
            else:
                self.compile_multi_model_trainer(X, y, training_cycles, **kwargs)
        for e in range(self.training_cycles):
            self.train_step()
            if any([e == 0, (e + 1) % kwargs.get("print_loss", 10) == 0,
                    e == self.training_cycles - 1]):
                self.print_statistics(e)
        return self.gp_model

    def save_weights(self, filename: str) -> None:
        """Saves weights of the feature extractor."""
        torch.save(self.gp_model.feature_extractor.state_dict(), filename)
