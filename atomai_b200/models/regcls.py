"""
Regressor (image -> vector) and Classifier (image -> class) with the MobileNetV2 backbone, drop-in
for atomai.models.Regressor / Classifier (atomai/models/regressor.py, classifier.py).  Training runs
the BaseTrainer loop (native forward / backward, fused loss and Adam, data parallelism under
torchrun); the networks are nets.RegressorNet / nets.ClassifierNet.
"""
from typing import Optional, Type, Union

import numpy as np
import torch

from ..predictors import RegPredictor, clsPredictor
from ..trainers import RegTrainer, clsTrainer
from ..transforms import reg_augmentor


def _load_weights(model, filepath: str) -> None:
    weight_dict = torch.load(filepath, map_location=model.device)
    if "weights" in weight_dict:
        weight_dict = weight_dict["weights"]
    model.net.load_state_dict(weight_dict)


class Regressor(RegTrainer):
    """
    Model for image -> vector regression

    Args:
        model: backbone ('mobilenet'; 'resnet' and 'vgg' raise NotImplementedError)
        out_dim: output dimensions (Default: 1)
        **input_channels: image channels (Default: 1)
        **seed: random seed (Default: 1)

    Example:
        >>> model = Regressor(out_dim=1)
        >>> model.fit(train_images, train_targets, test_images, test_targets,
        >>>           full_epoch=True, training_cycles=30, swa=True)
        >>> prediction = model.predict(imgs_new, norm=True)
    """
    def __init__(self, model: str = 'mobilenet', out_dim: int = 1, **kwargs) -> None:
        super(Regressor, self).__init__(out_dim, model, **kwargs)

    def fit(self,
            X_train: Union[np.ndarray, torch.Tensor],
            y_train: Union[np.ndarray, torch.Tensor],
            X_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            y_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            loss: str = 'mse',
            optimizer: Optional[Type[torch.optim.Optimizer]] = None,
            training_cycles: int = 1000,
            batch_size: int = 64,
            compute_accuracy: bool = False,
            full_epoch: bool = False,
            swa: bool = False,
            perturb_weights: bool = False,
            **kwargs):
        """
        Trains the model — arguments and kwargs (test_size, seed, print_loss, filename,
        lr_scheduler, batch_seed, memory_alloc and the image noise augmentations) as in
        atomai/models/regressor.py:34-111.
        """
        self.compile_trainer(
            (X_train, y_train, X_test, y_test),
            loss, optimizer, training_cycles, batch_size,
            compute_accuracy, full_epoch, swa, perturb_weights,
            **kwargs)
        self.augment_fn = reg_augmentor(**kwargs)
        _ = self.run()

    def predict(self, data: np.ndarray, **kwargs) -> np.ndarray:
        """
        Predicts the target vector of an image (h, w) or a batch (n, h, w) / (n, c, h, w)
        (**num_batches (10), **norm (True): min-max normalise, **verbose (True)).
        """
        use_gpu = self.device == 'cuda'
        return RegPredictor(self.net, self.output_size, use_gpu, **kwargs).run(data, **kwargs)

    def load_weights(self, filepath: str) -> None:
        """Loads a state_dict, or the 'weights' of a saved meta-state dictionary."""
        _load_weights(self, filepath)


class Classifier(clsTrainer):
    """
    Model for image classification

    Args:
        model: backbone ('mobilenet'; 'resnet' and 'vgg' raise NotImplementedError)
        nb_classes: number of classes (required)
        **input_channels: image channels (Default: 1)
        **seed: random seed (Default: 1)

    Example:
        >>> model = Classifier(nb_classes=4)
        >>> model.fit(train_images, train_labels, test_images, test_labels,
        >>>           full_epoch=True, training_cycles=30, swa=True)
        >>> prediction = model.predict(imgs_new, norm=True)
    """
    def __init__(self, model: str = 'mobilenet', nb_classes: int = None, **kwargs) -> None:
        if nb_classes is None:
            raise AssertionError(
                "You must specify a number of classes (nb_classes) for your classification model")
        super(Classifier, self).__init__(nb_classes, model, **kwargs)

    def fit(self,
            X_train: Union[np.ndarray, torch.Tensor],
            y_train: Union[np.ndarray, torch.Tensor],
            X_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            y_test: Optional[Union[np.ndarray, torch.Tensor]] = None,
            loss: str = 'nll',
            optimizer: Optional[Type[torch.optim.Optimizer]] = None,
            training_cycles: int = 1000,
            batch_size: int = 64,
            compute_accuracy: bool = False,
            full_epoch: bool = False,
            swa: bool = False,
            perturb_weights: bool = False,
            **kwargs):
        """
        Trains the model on images and 1-D int64 labels — arguments and kwargs as in
        atomai/models/classifier.py:37-116.  The criterion is always the mean NLL of the network's
        log-probabilities (`loss` is kept for the reference's signature).
        """
        self.compile_trainer(
            (X_train, y_train, X_test, y_test),
            loss, optimizer, training_cycles, batch_size,
            compute_accuracy, full_epoch, swa, perturb_weights,
            **kwargs)
        self.augment_fn = reg_augmentor(**kwargs)
        _ = self.run()

    def predict(self, data: np.ndarray, **kwargs) -> np.ndarray:
        """
        Predicts the class of an image (h, w) or a batch (n, h, w) / (n, c, h, w)
        (**num_batches (10), **norm (True): min-max normalise, **verbose (True)).
        """
        use_gpu = self.device == 'cuda'
        return clsPredictor(self.net, self.nb_classes, use_gpu, **kwargs).run(data, **kwargs)

    def load_weights(self, filepath: str) -> None:
        """Loads a state_dict, or the 'weights' of a saved meta-state dictionary."""
        _load_weights(self, filepath)
