"""
Inference wrappers and NN-output -> atom coordinates, with the reference's interface
(atomai/predictors/predictor.py:23-298, 531-639).  The network forward runs on the GPU (native
sm_90a graph) and so does the Locator's front end: one kernel turns the NHWC logits into class
probabilities AND the thresholded binary masks (atomai_b200_prob_mask), batches are copied to
pinned host buffers asynchronously and synchronised once.  Connected components -> centre of mass
-> edge filter stay the reference's CPU algorithm (scipy.ndimage) on those masks, bit-exact with
the reference (tests/golden/locator_crop.npz, bfo_1024.npz).
"""
import time
from typing import Dict, List, Tuple, Type, Union

import numpy as np
import torch

from ..utils.coords import find_com
from ..utils.img import cv_thresh, img_pad, img_resize
from ..utils.nn import get_downsample_factor, get_nb_classes, set_train_rng
from ..utils.preproc import torch_format_image, torch_format_spectra


class BasePredictor:
    """Base predictor class (atomai/predictors/predictor.py:23-121)."""
    def __init__(self, model: Type[torch.nn.Module] = None, use_gpu: bool = False,
                 **kwargs: Union[bool, str]) -> None:
        self.model = model
        self.device = "cpu"
        if use_gpu and torch.cuda.is_available():
            self.device = kwargs.get("device") or "cuda"
        if self.model is not None:
            self.model.to(self.device)
        self.verbose = kwargs.get("verbose", False)

    def preprocess(self, data: Union[torch.Tensor, np.ndarray]) -> torch.Tensor:
        if isinstance(data, np.ndarray):
            data = torch.from_numpy(data).float()
        return data

    def _model2device(self, device: str = None) -> None:
        self.model.to(self.device if device is None else device)

    def _data2device(self, data: torch.Tensor, device: str = None) -> torch.Tensor:
        return data.to(self.device if device is None else device)

    def forward_(self, xnew: torch.Tensor) -> torch.Tensor:
        self.model.eval()
        with torch.no_grad():
            out = self.model(xnew.to(self.device))
        return out

    def batch_predict(self, data: torch.Tensor, out_shape: Tuple[int],
                      num_batches: int) -> torch.Tensor:
        """Batch-by-batch prediction into a CPU tensor (predictor.py:82-106)."""
        batch_size = len(data) // num_batches
        if batch_size < 1:
            num_batches = batch_size = 1
        prediction_all = torch.zeros(out_shape)
        stop = num_batches * batch_size
        for i in range(num_batches):
            if self.verbose:
                print("\rBatch {}/{}".format(i + 1, num_batches), end="")
            sl = slice(i * batch_size, (i + 1) * batch_size)
            prediction_all[sl] = self.forward_(data[sl]).cpu()
        if len(data) > stop:
            prediction_all[stop:] = self.forward_(data[stop:]).cpu()
        return prediction_all

    def predict(self, data: torch.Tensor, out_shape: Tuple[int] = None,
                num_batches: int = 1) -> torch.Tensor:
        out_shape = data.shape if out_shape is None else (data.shape[0], *out_shape)
        data = self.preprocess(data)
        return self.batch_predict(data, out_shape, num_batches)


class SegPredictor(BasePredictor):
    """
    Prediction with a trained fully convolutional neural network; arguments as in
    atomai/predictors/predictor.py:124-188 (trained_model, refine, resize, use_gpu, logits,
    **thresh, **d, **nb_classes, **downsampling).

    Example:
        >>> nn_output, coords = SegPredictor(trained_model, use_gpu=True).run(expdata)
    """
    def __init__(self, trained_model: Type[torch.nn.Module], refine: bool = False,
                 resize: Union[Tuple, List] = None, use_gpu: bool = False, logits: bool = True,
                 **kwargs: Union[int, float, bool]) -> None:
        super(SegPredictor, self).__init__(trained_model, use_gpu)
        set_train_rng(1)
        self.nb_classes = kwargs.get('nb_classes', None)
        if self.nb_classes is None:
            self.nb_classes = get_nb_classes(trained_model)
        self.downsampling = kwargs.get('downsampling', None)
        if self.downsampling is None:
            self.downsampling = get_downsample_factor(trained_model)
        self.resize = resize
        self.logits = logits
        self.refine = refine
        self.d = kwargs.get("d", None)
        self.thresh = kwargs.get("thresh", .5)
        self.use_gpu = use_gpu
        self.verbose = kwargs.get("verbose", True)

    def preprocess(self, image_data: np.ndarray, norm: bool = True) -> torch.Tensor:
        """squeeze channel dim, optional resize, pad to the downsampling factor, global min-max
        normalisation in float64 -> float32 (predictor.py:190-207)."""
        if image_data.ndim == 2:
            image_data = image_data[np.newaxis, ...]
        elif image_data.ndim == 4:
            if image_data.shape[-1] == 1:
                image_data = image_data[..., 0]
            elif image_data.shape[1] == 1:
                image_data = image_data[:, 0, ...]
        if self.resize is not None:
            image_data = img_resize(image_data, self.resize)
        image_data = img_pad(image_data, self.downsampling)
        return torch_format_image(image_data, norm)

    def _prob_mode(self) -> int:
        """softmax / sigmoid for raw logits, exp for log-probabilities (predictor.py:219-228)."""
        if self.logits:
            return 0 if self.nb_classes > 1 else 1
        return 2 if self.nb_classes > 1 else 3

    def forward_device(self, images: torch.Tensor, with_mask: bool = True):
        """Network forward + fused probability / threshold kernel; returns channel-last device
        tensors (prob fp32 (n,h,w,c), mask uint8 (n,h,w,c) or None)."""
        from .. import ops
        images = images.to(self.device, non_blocking=True)
        self.model.eval()
        with torch.no_grad():
            logits = self.model(images)
        lg = logits.permute(0, 2, 3, 1)
        if not lg.is_contiguous():
            lg = lg.contiguous()
        prob = torch.empty(lg.shape, device=lg.device, dtype=torch.float32)
        mask = torch.empty(lg.shape, device=lg.device, dtype=torch.uint8) if with_mask else None
        ops.prob_mask(lg, self._prob_mode(), self.thresh, prob, mask)
        return prob, mask

    def forward_(self, images: torch.Tensor) -> torch.Tensor:
        """Per-pixel class 'probabilities', channel-last, on the CPU (predictor.py:209-231)."""
        return self.forward_device(images, with_mask=False)[0].cpu()

    def batch_predict(self, data: torch.Tensor, out_shape: Tuple[int],
                      num_batches: int) -> torch.Tensor:
        """Batch-by-batch prediction (predictor.py:82-106) without a host sync per batch: every
        batch's probabilities and masks are copied into pinned host buffers on the compute stream
        and the host waits once at the end.  The masks are kept in `self.masks_`."""
        if self.device == "cpu" or not torch.cuda.is_available():
            raise RuntimeError("atomai_b200 predicts on CUDA (sm_90a) only; there is no CPU path")
        batch_size = len(data) // num_batches
        if batch_size < 1:
            num_batches = batch_size = 1
        prediction_all = torch.zeros(out_shape).pin_memory()
        masks_all = torch.zeros(out_shape, dtype=torch.uint8).pin_memory()
        stop = num_batches * batch_size
        bounds = [(i * batch_size, (i + 1) * batch_size) for i in range(num_batches)]
        if len(data) > stop:
            bounds.append((stop, len(data)))
        for i, (b0, b1) in enumerate(bounds):
            if self.verbose:
                print("\rBatch {}/{}".format(min(i + 1, num_batches), num_batches), end="")
            prob, mask = self.forward_device(data[b0:b1])
            prediction_all[b0:b1].copy_(prob, non_blocking=True)
            masks_all[b0:b1].copy_(mask, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.masks_ = masks_all.numpy()
        return prediction_all

    def predict(self, image_data: np.ndarray, return_image: bool = False,
                **kwargs: int) -> Tuple[np.ndarray]:
        """Make prediction (predictor.py:233-262): one image per batch for >= 256 px frames,
        otherwise 10 batches, unless num_batches is given."""
        image_data = self.preprocess(image_data, kwargs.get("norm", True))
        n, _, w, h = image_data.shape
        num_batches = kwargs.get("num_batches")
        if num_batches is None:
            num_batches = len(image_data) if (w >= 256 or h >= 256) else 10
        segmented_imgs = self.batch_predict(image_data, (n, w, h, self.nb_classes), num_batches)
        if return_image:
            return image_data.permute(0, 2, 3, 1).numpy(), segmented_imgs.numpy()
        return segmented_imgs.numpy()

    def run(self, image_data: np.ndarray, compute_coords=True,
            **kwargs: int) -> Tuple[np.ndarray, Dict[int, np.ndarray]]:
        """Prediction + coordinates (predictor.py:264-298)."""
        start_time = time.time()
        if not compute_coords:
            return self.predict(image_data, **kwargs)
        if "thresh" in kwargs:
            self.thresh = kwargs["thresh"]
        images, decoded_imgs = self.predict(image_data, return_image=True, **kwargs)
        loc = Locator(self.thresh, refine=self.refine, d=self.d)
        coordinates = loc.run(decoded_imgs, images, masks=getattr(self, "masks_", None))
        if self.verbose:
            n_images_str = " image was " if decoded_imgs.shape[0] == 1 else " images were "
            print("\n" + str(decoded_imgs.shape[0]) + n_images_str +
                  "decoded in approximately " +
                  str(np.around(time.time() - start_time, decimals=4)) + ' seconds')
        return decoded_imgs, coordinates


class ImSpecPredictor(BasePredictor):
    """
    Prediction with a trained im2spec / spec2im model (atomai/predictors/predictor.py:301-395).

    Args:
        trained_model: trained SignalED network
        output_dim: (length,) for im2spec, (height, width) for spec2im
        use_gpu: the native kernels need CUDA; the flag is kept for signature parity
        **verbose (bool)

    Example:
        >>> prediction = ImSpecPredictor(trained_model, (16,), use_gpu=True).run(data)
    """
    def __init__(self, trained_model: Type[torch.nn.Module], output_dim: Tuple[int],
                 use_gpu: bool = False, **kwargs: str) -> None:
        super(ImSpecPredictor, self).__init__(trained_model, use_gpu)
        if isinstance(output_dim, int):
            output_dim = (output_dim,)
        if len(output_dim) not in [1, 2]:
            raise ValueError("output_dim must be a two-value tuple for images" +
                             " and a single-value tuple for spectra")
        set_train_rng(1)
        self.output_dim = output_dim
        self.verbose = kwargs.get("verbose", True)

    def preprocess(self, signal: np.ndarray, norm: bool = True) -> torch.Tensor:
        """Adds the batch / channel axes and (optionally) scales to (0, 1)."""
        if len(self.output_dim) == 1:
            if signal.ndim == 2:
                signal = signal[np.newaxis, ...]
            signal = torch_format_image(signal, norm)
        elif len(self.output_dim) == 2:
            if signal.ndim == 1:
                signal = signal[np.newaxis, ...]
            signal = torch_format_spectra(signal, norm)
        return signal

    def predict(self, signal: np.ndarray, **kwargs: int) -> np.ndarray:
        """Spectra from images or vice versa; **num_batches (default 10), **norm (default True)."""
        signal = self.preprocess(signal, kwargs.get("norm", True))
        num_batches = kwargs.get("num_batches", 10)
        output = self.batch_predict(signal, (len(signal), 1, *self.output_dim), num_batches)
        return output[:, 0].numpy()

    def run(self, signal: np.ndarray, **kwargs: int) -> np.ndarray:
        """predict + the reference's timing line."""
        start_time = time.time()
        prediction = self.predict(signal, **kwargs)
        if self.verbose:
            if len(self.output_dim) == 1:
                str_ = " image was " if prediction.shape[0] == 1 else " images were "
            else:
                str_ = " spectrum was " if prediction.shape[0] == 1 else " spectra were "
            print("\n" + str(prediction.shape[0]) + str_ + "decoded in approximately "
                  + str(np.around(time.time() - start_time, decimals=4)) + ' seconds')
        return prediction


class Locator:
    """
    Transforms pixel data from NN output into coordinate data
    (atomai/predictors/predictor.py:531-639): threshold -> 4-connected components -> centre of
    mass (of the thresholded image) -> drop coordinates within `dist_edge` px of the border.
    Returns {frame: (n_atoms, 3) float64 [x, y, class]}.

    Example:
        >>> coordinates = Locator(dist_edge=10, refine=False).run(nn_output)
    """
    def __init__(self, threshold: float = 0.5, dist_edge: int = 5,
                 dim_order: str = 'channel_last', **kwargs: Union[bool, float]) -> None:
        self.dim_order = dim_order
        self.threshold = threshold
        self.dist_edge = dist_edge
        self.refine = kwargs.get("refine")
        self.d = kwargs.get("d")

    def preprocess(self, nn_output: np.ndarray) -> np.ndarray:
        if nn_output.shape[-1] == 1:   # add the background class for 1-channel data
            nn_output = np.concatenate((nn_output, 1 - nn_output), axis=3)
        if self.dim_order == 'channel_first':
            nn_output = np.transpose(nn_output, (0, 2, 3, 1))
        elif self.dim_order != 'channel_last':
            raise NotImplementedError('For dim_order, use "channel_first"',
                                      'or "channel_last" (e.g. tensorflow)')
        return nn_output

    def run(self, nn_output: np.ndarray, *args: np.ndarray,
            masks: np.ndarray = None) -> Dict[int, np.ndarray]:
        """`masks` (optional, uint8 (n,h,w,c), channel-last): the binary images `nn_output >
        threshold` already computed on the GPU by SegPredictor; otherwise thresholded here."""
        nn_output = self.preprocess(nn_output)
        h, w = nn_output.shape[1:3]
        if masks is not None and (self.dim_order != 'channel_last' or
                                  masks.shape[:3] != nn_output.shape[:3]):
            masks = None
        d_coord = {}
        for i, decoded_img in enumerate(nn_output):
            per_class = []
            for ch in range(decoded_img.shape[2] - 1):   # background is always the last class
                if masks is not None and ch < masks.shape[3]:
                    blobs = masks[i, :, :, ch].astype(decoded_img.dtype)
                else:
                    blobs = cv_thresh(decoded_img[:, :, ch], self.threshold)
                coord_ch = self.rem_edge_coord(find_com(blobs), h, w)
                per_class.append(np.concatenate(
                    (coord_ch, np.zeros((coord_ch.shape[0], 1)) + ch), axis=1))
            d_coord[i] = np.concatenate(per_class, axis=0) if per_class else np.empty((0, 3))
        if self.refine:
            raise NotImplementedError(
                "2-D Gaussian peak refinement (atomai/utils/coords.py:179-231) is outside the "
                "accelerated hot path; pass refine=False")
        return d_coord

    def rem_edge_coord(self, coordinates: np.ndarray, h: int, w: int) -> np.ndarray:
        """Removes coordinates at the image edges (predictor.py:622-639)."""
        if coordinates.shape[0] == 0:
            return coordinates
        e = self.dist_edge
        bad = ((coordinates[:, 0] > h - e) | (coordinates[:, 0] < e) |
               (coordinates[:, 1] > w - e) | (coordinates[:, 1] < e))
        return coordinates[~bad]
