"""
Deep-ensemble training with the reference's interface (atomai/trainers/etrainer.py:29-512):
BaseEnsembleTrainer / EnsembleTrainer with train_baseline, train_ensemble_from_scratch,
train_ensemble_from_baseline, train_swag, save_ensemble_metadict.  Every member is an ordinary
BaseTrainer run on the native sm_90a path.

Multi-GPU (new; the reference is single-device): ensembles are the "replicas" workload of
SURVEY.md §8e/§8f — members are independent, so under torchrun member i is trained by rank
i mod world on its own GPU with NO data-path collective (data parallelism is switched off for
these runs) and the trained state_dicts are exchanged once at the end.
"""
import warnings
from copy import deepcopy as dc
from typing import Callable, Dict, Optional, Tuple, Type, Union

import numpy as np
import torch

from ..nets import init_fcnn_model, init_imspec_model
from ..utils.nn import average_weights, sample_weights
from ..utils.preproc import check_image_dims, check_signal_dims, num_classes_from_labels
from .trainer import BaseTrainer

augfn_type = Callable[[torch.Tensor, torch.Tensor, int], Tuple[torch.Tensor, torch.Tensor]]
ensemble_type = Dict[int, Dict[str, torch.Tensor]]


def _dist():
    d = torch.distributed
    if d.is_available() and d.is_initialized() and d.get_world_size() > 1:
        return d.get_rank(), d.get_world_size()
    return 0, 1


class BaseEnsembleTrainer(BaseTrainer):
    """Base class for deep ensemble training (etrainer.py:29-298)."""
    def __init__(self, model: Type[torch.nn.Module] = None, nb_classes=None) -> None:
        super(BaseEnsembleTrainer, self).__init__()
        self._no_dp = True            # members are replicas: no gradient all-reduce between ranks
        if model is not None:
            self.set_model(model, nb_classes)
        self.ensemble_state_dict = {}
        self.kdict = {}

    def compile_ensemble_trainer(self, **kwargs) -> None:
        """kwargs are passed on to BaseTrainer.compile_trainer (loss, optimizer, full_epoch, swa,
        perturb_weights, batch_size, training_cycles, filename, print_loss, ...)."""
        self.kdict = kwargs

    def train_baseline(self, X_train, y_train, X_test=None, y_test=None, seed: int = 1,
                       augment_fn: augfn_type = None) -> Type[torch.nn.Module]:
        """Trains baseline weights from a fresh initialisation (etrainer.py:60-103)."""
        if self.net is None:
            raise AssertionError("You need to set a model first")
        self._reset_rng(seed)
        self._reset_weights()
        self._reset_training_history()
        self._delete_optimizer()
        (X_train, y_train, X_test, y_test) = self.preprocess_train_data(
            X_train, y_train, X_test, y_test)
        self.compile_trainer((X_train, y_train, X_test, y_test), **self.kdict)
        self.data_augmentation(augment_fn)
        self.fit()
        return self.net

    def _gather_members(self, mine: Dict[int, dict]) -> None:
        """Every rank ends up with every member's weights (one object all-gather, CPU tensors)."""
        rank, world = _dist()
        if world == 1:
            self.ensemble_state_dict.update(mine)
            return
        cpu = {i: {k: v.cpu() for k, v in sd.items()} for i, sd in mine.items()}
        out = [None] * world
        torch.distributed.all_gather_object(out, cpu)
        for part in out:
            for i, sd in part.items():
                self.ensemble_state_dict[i] = {k: v.to(self.device) for k, v in sd.items()}
        self.ensemble_state_dict = dict(sorted(self.ensemble_state_dict.items()))

    def train_ensemble_from_scratch(self, X_train, y_train, X_test=None, y_test=None,
                                    n_models: int = 10, augment_fn: augfn_type = None, **kwargs
                                    ) -> Tuple[Type[torch.nn.Module], ensemble_type]:
        """Trains `n_models` models, each from a different initialisation (seed = member index)
        and batch order (etrainer.py:105-149).  Returns the last model trained on this rank and
        the dictionary with all ensemble weights."""
        self.update_training_parameters(kwargs)
        rank, world = _dist()
        if self._is_main():
            print("Training ensemble models (strategy = 'from_scratch')")
        mine = {}
        for i in range(rank, n_models, world):
            print("\nEnsemble model {}".format(i + 1))
            self.kdict["batch_seed"] = i
            model_i = self.train_baseline(X_train, y_train, X_test, y_test, i, augment_fn)
            mine[i] = dc(model_i.state_dict())
        self._gather_members(mine)
        self.save_ensemble_metadict()
        return self.net, self.ensemble_state_dict

    def train_ensemble_from_baseline(self, X_train, y_train, X_test=None, y_test=None,
                                     basemodel: Type[torch.nn.Module] = None, n_models: int = 10,
                                     training_cycles_base: int = 1000,
                                     training_cycles_ensemble: int = 100,
                                     augment_fn: augfn_type = None, **kwargs
                                     ) -> Tuple[Type[torch.nn.Module], ensemble_type]:
        """Trains a baseline for N cycles (unless given), then `n_models` members for n << N cycles
        each from that baseline with different batch shuffling (etrainer.py:151-231).  Returns the
        model with averaged weights and the dictionary with ensemble weights."""
        self.update_training_parameters(kwargs)
        rank, world = _dist()
        if basemodel is None:
            self.kdict["training_cycles"] = training_cycles_base
            if self._is_main():
                print("Training baseline model...")
            basemodel = self.train_baseline(X_train, y_train, X_test, y_test, 1, augment_fn)
        else:
            (X_train, y_train, X_test, y_test) = self.preprocess_train_data(
                X_train, y_train, X_test, y_test)
        self.set_model(basemodel)
        basemodel_state_dict = dc(self.net.state_dict())
        self.kdict["training_cycles"] = training_cycles_ensemble
        if not self.full_epoch and "print_loss" not in self.kdict.keys():
            self.kdict["print_loss"] = 10
        if self._is_main():
            print("\nTraining ensemble models (strategy = 'from_baseline')")
        mine = {}
        model_i = self.net
        for i in range(rank, n_models, world):
            print("\nEnsemble model {}".format(i + 1))
            self.net.load_state_dict(basemodel_state_dict)
            self._reset_rng(i + 2)
            self._reset_training_history()
            self._delete_optimizer()
            kd = dict(self.kdict)
            kd["batch_seed"] = i + 2
            self.compile_trainer((X_train, y_train, X_test, y_test), **kd)
            model_i = self.run()
            mine[i] = dc(model_i.state_dict())
        self._gather_members(mine)
        self.save_ensemble_metadict()
        model_i.load_state_dict(average_weights(self.ensemble_state_dict))
        return model_i, self.ensemble_state_dict

    def train_swag(self, X_train, y_train, X_test=None, y_test=None, n_models: int = 10,
                   augment_fn: augfn_type = None, **kwargs
                   ) -> Tuple[Type[torch.nn.Module], ensemble_type]:
        """SWAG-like weight sampling at the end of a single training run (etrainer.py:233-269)."""
        self.update_training_parameters(kwargs)
        self.kdict["swa"] = True
        basemodel = self.train_baseline(X_train, y_train, X_test, y_test, 1, augment_fn)
        self.ensemble_state_dict = sample_weights(self.running_weights, n_models)
        self.save_ensemble_metadict()
        return basemodel, self.ensemble_state_dict

    def update_training_parameters(self, kwargs):
        warn_msg = "Overwriting the initial value '{}' of parameter '{}' with new value '{}'"
        for k, v in kwargs.items():
            if k in self.kdict.keys():
                warnings.warn(warn_msg.format(self.kdict[k], k, kwargs[k]), UserWarning)
            self.kdict[k] = v

    def preprocess_train_data(self, *train_data) -> Tuple[torch.Tensor]:
        tor = lambda x: torch.from_numpy(x) if isinstance(x, np.ndarray) else x  # noqa: E731
        return tuple(tor(x) for x in train_data)

    def save_ensemble_metadict(self, filename: str = None) -> None:
        """Saves the meta dictionary with the ensemble weights as <filename>_ensemble_metadict.tar
        (etrainer.py:290-298); rank 0 only."""
        if not self._is_main():
            return
        fname = self.filename if filename is None else filename
        ensemble_metadict = {k: v for k, v in self.meta_state_dict.items()
                             if k not in ("weights", "optimizer")}
        ensemble_metadict["weights"] = self.ensemble_state_dict
        torch.save(ensemble_metadict, fname + "_ensemble_metadict.tar")


class EnsembleTrainer(BaseEnsembleTrainer):
    """
    Deep ensemble trainer (etrainer.py:301-433).

    Args: model ('Unet', 'dilnet', 'imspec' or an initialised torch module), nb_classes and the
    model kwargs (for 'imspec': in_dim, out_dim, latent_dim).

    Example:

        >>> etrainer = EnsembleTrainer("Unet", batch_norm=True, nb_classes=3)
        >>> etrainer.compile_ensemble_trainer(training_cycles=500)
        >>> smodel, ensemble = etrainer.train_ensemble_from_scratch(
        >>>    images, labels, images_test, labels_test, n_models=10)
    """
    def __init__(self, model: Union[str, Type[torch.nn.Module]] = None, nb_classes: int = 1,
                 **kwargs) -> None:
        super(EnsembleTrainer, self).__init__()
        self.nb_classes = nb_classes
        if isinstance(model, str):
            if model in ["Unet", "dilnet", "SegResNet", "ResHedNet"]:
                self.net, self.meta_state_dict = init_fcnn_model(model, self.nb_classes, **kwargs)
            elif model == "imspec":
                missing = [k for k in ["in_dim", "out_dim", "latent_dim"] if k not in kwargs]
                if missing:
                    raise AssertionError("Specify input, output, and latent dimensions " +
                                         "(Missing dimensions: {})".format(str(missing)[1:-1]))
                self.in_dim, self.out_dim = kwargs.pop("in_dim"), kwargs.pop("out_dim")
                latent_dim = kwargs.pop("latent_dim")
                self.net, self.meta_state_dict = init_imspec_model(
                    self.in_dim, self.out_dim, latent_dim, **kwargs)
            else:
                raise NotImplementedError(f"unknown model '{model}'")
            self.net.to(self.device)
        else:
            self.set_model(model, nb_classes)
        self.meta_state_dict["weights"] = self.net.state_dict()
        self.meta_state_dict["optimizer"] = self.optimizer

    def compile_ensemble_trainer(self, **kwargs) -> None:
        self.kdict = kwargs
        self.full_epoch = self.kdict.get("full_epoch", False)
        self.batch_size = self.kdict.get("batch_size", 32)
        self.kdict["overwrite_train_data"] = False

    def train_baseline(self, X_train, y_train, X_test=None, y_test=None, seed: int = 1,
                       augment_fn: augfn_type = None) -> Type[torch.nn.Module]:
        if self.net is None:
            raise AssertionError("You need to set a model first")
        train_data = self.preprocess_train_data(X_train, y_train, X_test, y_test)
        self.set_data(*train_data, **{k: v for k, v in self.kdict.items() if k == "memory_alloc"})
        self._reset_rng(seed)
        self._reset_weights()
        self._reset_training_history()
        self._delete_optimizer()
        self.compile_trainer((X_train, y_train, X_test, y_test), **self.kdict)
        self.data_augmentation(augment_fn)
        self.fit()
        return self.net

    def preprocess_train_data(self, *args: np.ndarray) -> Tuple[np.ndarray]:
        """Training and test data preprocessing (etrainer.py:424-433)."""
        if self.meta_state_dict.get("model_type") == "seg":
            return set_data_seg(*args, self.nb_classes)
        if self.meta_state_dict.get("model_type") == "imspec":
            return set_data_imspec(*args, (self.in_dim, self.out_dim))
        return tuple(args)


def set_data_seg(X_train, y_train, X_test=None, y_test=None, nb_classes_set: int = 1, **kwargs):
    """Sets training and test data for semantic segmentation (etrainer.py:436-467)."""
    nb_classes = num_classes_from_labels(y_train)
    if nb_classes != nb_classes_set:
        raise AssertionError("Number of specified classes" +
                             " is different from the number of classes" +
                             " contained in training data")
    if X_test is None or y_test is None:
        from sklearn.model_selection import train_test_split
        X_train, X_test, y_train, y_test = train_test_split(
            X_train, y_train, test_size=kwargs.get("test_size", .15),
            shuffle=True, random_state=kwargs.get("seed", 1))
    X_train, y_train, X_test, y_test = check_image_dims(X_train, y_train, X_test, y_test, nb_classes)
    f32, i64 = lambda x: x.astype(np.float32), lambda x: x.astype(np.int64)  # noqa: E731
    X_train, X_test = f32(X_train), f32(X_test)
    if nb_classes > 1:
        y_train, y_test = i64(y_train), i64(y_test)
    else:
        y_train, y_test = f32(y_train), f32(y_test)
    return X_train, y_train, X_test, y_test


def set_data_imspec(X_train, y_train, X_test=None, y_test=None, dims=None, **kwargs):
    """Sets training and test data for im2spec / spec2im models (etrainer.py:470-499)."""
    if X_test is None or y_test is None:
        from sklearn.model_selection import train_test_split
        X_train, X_test, y_train, y_test = train_test_split(
            X_train, y_train, test_size=kwargs.get("test_size", .15),
            shuffle=True, random_state=kwargs.get("seed", 1))
    X_train, y_train, X_test, y_test = check_signal_dims(X_train, y_train, X_test, y_test)
    in_dim, out_dim = X_train.shape[2:], y_train.shape[2:]
    if tuple(dims[0]) != tuple(in_dim) or tuple(dims[1]) != tuple(out_dim):
        raise AssertionError("The input/output dimensions of the model must match" +
                             " the height, width and length (for spectra) of training")
    f32 = lambda x: x.astype(np.float32)  # noqa: E731
    return f32(X_train), f32(y_train), f32(X_test), f32(y_test)
