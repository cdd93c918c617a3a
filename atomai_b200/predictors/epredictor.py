"""
Prediction with an ensemble of models (atomai/predictors/epredictor.py:21-267): EnsemblePredictor
(mean and variance over the members' outputs) and ensemble_locate.  Every member's forward runs on
the native sm_90a graph; the running mean / M2 accumulation over members stays on the device, so
only the final mean and variance cross PCIe (the reference copies every member's full output).
"""
from typing import Dict, Tuple, Type, Union

import numpy as np
import torch

from ..utils.nn import get_downsample_factor
from ..utils.preproc import torch_format_image, torch_format_spectra
from .predictor import BasePredictor, Locator


class EnsemblePredictor(BasePredictor):
    """
    Prediction with ensemble of models

    Args: skeleton (model with the ensemble's architecture), ensemble ({i: state_dict}), data_type
    / output_type ('image' | 'spectra'), nb_classes, in_dim, out_dim, **output_shape, **verbose,
    **logits, **use_gpu — epredictor.py:21-84.

    Example:
        >>> p = EnsemblePredictor(skeleton, ensemble, nb_classes=3)
        >>> nn_out_mean, nn_out_var = p.predict(expdata)
    """
    def __init__(self, skeleton: Type[torch.nn.Module], ensemble: Dict[int, Dict[str, torch.Tensor]],
                 data_type: str = "image", output_type: str = "image", nb_classes: int = None,
                 in_dim: Tuple[int] = None, out_dim: Tuple[int] = None,
                 **kwargs: Union[str, Tuple[int]]) -> None:
        super(EnsemblePredictor, self).__init__()
        if output_type not in ["image", "spectra"]:
            raise TypeError("Supported output types are 'image' and 'spectra'")
        inout = [data_type, output_type]
        if inout in (["image", "spectra"], ["spectra", "image"]) and not all([in_dim, out_dim]):
            raise TypeError("Specify input (in_dim) & output (out_dim) dimensions")
        if not torch.cuda.is_available():
            raise RuntimeError("atomai_b200 predicts on CUDA (sm_90a) only; there is no CPU path")
        self.device = kwargs.get("device") or "cuda"
        self.model = skeleton
        self.ensemble = ensemble
        self.data_type, self.output_type = data_type, output_type
        self.nb_classes = nb_classes
        self.in_dim, self.out_dim = in_dim, out_dim
        self.downsample_factor = None
        self.logits = kwargs.get("logits", True)
        self.output_shape = kwargs.get("output_shape")
        verbose = kwargs.get("verbose", 1)
        self.everbose = bool(verbose)
        self.verbose = verbose > 1

    def _set_output_shape(self, data: np.ndarray) -> None:
        if self.data_type == self.output_type == "image":
            out_shape = (len(data), self.nb_classes if self.nb_classes else 1, *data.shape[2:])
        elif self.data_type == "spectra" and self.output_type == "image":
            out_shape = (len(data), self.nb_classes if self.nb_classes else 1, *self.out_dim)
        elif self.data_type == "image" and self.output_type == "spectra":
            out_shape = (len(data), 1, *self.out_dim)
        elif self.data_type == self.output_type == "spectra":
            out_shape = (len(data), 1, *data.shape[2:])
        else:
            raise TypeError("Data not understood")
        self.output_shape = out_shape

    def preprocess(self, data: np.ndarray, norm: bool = True) -> torch.Tensor:
        if self.data_type == "image":
            if data.ndim == 2:
                data = data[np.newaxis, ...]
            data = torch_format_image(data, norm)
        elif self.data_type == "spectra":
            if data.ndim == 1:
                data = data[np.newaxis, ...]
            data = torch_format_spectra(data, norm)
        return data

    def _member_prob(self, data_dev: torch.Tensor) -> torch.Tensor:
        with torch.no_grad():
            prob = self.model(data_dev)
        ncls = 0 if not self.nb_classes else self.nb_classes
        if self.logits:
            if ncls > 1:
                prob = torch.softmax(prob, dim=1)
            elif self.nb_classes == 1:
                prob = torch.sigmoid(prob)
        elif ncls > 1:
            prob = torch.exp(prob)
        return prob

    def ensemble_forward(self, data: torch.Tensor, out_shape: Tuple[int] = None,
                         num_batches: int = 1) -> np.ndarray:
        """ALL members' predictions, (n_models, n_samples, ...) — epredictor.py:132-161."""
        data_dev = data.to(self.device)
        self.model.to(self.device).eval()
        out = []
        for m in self.ensemble.values():
            self.model.load_state_dict(m)
            out.append(self._member_prob(data_dev).cpu().numpy())
        return np.stack(out).astype(np.float64)

    def ensemble_forward_(self, data: torch.Tensor, out_shape: Tuple[int] = None
                          ) -> Tuple[np.ndarray]:
        """Mean and (population) variance over the members, accumulated on the device in float64
        (Welford), equal to np.mean / np.var of the stacked member outputs."""
        data_dev = data.to(self.device)
        self.model.to(self.device).eval()
        mean = m2 = None
        for k, m in enumerate(self.ensemble.values(), 1):
            self.model.load_state_dict(m)
            p = self._member_prob(data_dev).double()
            if mean is None:
                mean, m2 = p.clone(), torch.zeros_like(p)
            else:
                d = p - mean
                mean += d / k
                m2 += d * (p - mean)
        return mean.cpu().numpy(), (m2 / len(self.ensemble)).cpu().numpy()

    def ensemble_batch_predict(self, data: torch.Tensor, num_batches: int = 10
                               ) -> Tuple[np.ndarray]:
        """Batch-by-batch prediction with ensemble models (epredictor.py:163-189)."""
        batch_size = len(data) // num_batches
        if batch_size < 1:
            num_batches = batch_size = 1
        prediction_mean = np.zeros(shape=self.output_shape)
        prediction_var = np.zeros(shape=self.output_shape)
        bounds = [(i * batch_size, (i + 1) * batch_size) for i in range(num_batches)]
        if len(data) > num_batches * batch_size:
            bounds.append((num_batches * batch_size, len(data)))
        for i, (b0, b1) in enumerate(bounds):
            if self.everbose:
                print("\rBatch {}/{}".format(min(i + 1, num_batches), num_batches), end="")
            prediction_mean[b0:b1], prediction_var[b0:b1] = self.ensemble_forward_(data[b0:b1])
        return prediction_mean, prediction_var

    def predict(self, data: np.ndarray, num_batches: int = 10, format_out: str = "channel_last",
                norm: bool = True) -> Tuple[np.ndarray]:
        """Mean and variance for all the data points with the ensemble (epredictor.py:191-235)."""
        if format_out not in ["channel_first", "channel_last"]:
            raise ValueError("Specify channel_last or channel_first output format")
        data = self.preprocess(data, norm)
        if not self.output_shape:
            self._set_output_shape(data)
        if self.data_type == self.output_type == "image" and self.downsample_factor is None:
            self.downsample_factor = get_downsample_factor(self.model)
        prediction_mean, prediction_var = self.ensemble_batch_predict(data, num_batches)
        if format_out == "channel_last":
            c_tr = (0, *(np.arange(prediction_mean.ndim - 2) + 2), 1)
        else:
            c_tr = np.arange(prediction_mean.ndim)
        return prediction_mean.transpose(c_tr), prediction_var.transpose(c_tr)


def cluster_coord(coord_class_dict, eps: float, min_samples: int = 10):
    """Collapses the coordinates of a stack onto the xy plane and clusters them with DBSCAN
    (atomai/utils/coords.py:304-347): returns (points per cluster, cluster means, cluster
    variances); like the reference, the first entry of np.unique(labels) is skipped."""
    from sklearn import cluster
    coordinates_all = np.empty((0, 3))
    for k in range(len(coord_class_dict)):
        coordinates_all = np.append(coordinates_all, coord_class_dict[k], axis=0)
    labels = cluster.DBSCAN(eps=eps, min_samples=min_samples).fit(coordinates_all[:, :2]).labels_
    clusters, clusters_var, clusters_mean = [], [], []
    for lab in np.unique(labels)[1:]:
        coord = coordinates_all[np.where(labels == lab)]
        clusters.append(coord)
        clusters_mean.append(np.mean(coord[:, :2], axis=0))
        clusters_var.append(np.var(coord[:, :2], axis=0))
    return clusters, np.array(clusters_mean), np.array(clusters_var)


def ensemble_locate(nn_output_ensemble: np.ndarray, **kwargs: Dict) -> Tuple[np.ndarray]:
    """Coordinates for each ensemble member's prediction and their per-atom mean / variance
    (atomai/predictors/epredictor.py:238-267): nn_output_ensemble is (n_models, n_images, h, w,
    c); kwargs eps (DBSCAN radius, default 0.5), threshold (Locator threshold, default 0.5)."""
    eps = kwargs.get("eps", 0.5)
    thresh = kwargs.get("threshold", 0.5)
    coord_mean_all, coord_var_all = {}, {}
    for i in range(nn_output_ensemble.shape[1]):
        coordinates = {}
        for i2, img in enumerate(nn_output_ensemble[:, i]):
            coordinates[i2] = Locator(thresh).run(img[None, ...])[0]
        _, coord_mean, coord_var = cluster_coord(coordinates, eps)
        coord_mean_all[i] = coord_mean
        coord_var_all[i] = coord_var
    return coord_mean_all, coord_var_all
