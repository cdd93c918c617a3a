"""
On-the-fly data augmentation on the GPU — the reference's `datatransform` / `seg_augmentor` /
`imspec_augmentor` (atomai/transforms/imaug.py:20-478) without the device -> host -> device round
trip it makes every training step.  Supported, in the reference's order: rotation (flips / 90
degree turns, images AND label maps), gauss_noise, jitter, poisson_noise, salt_and_pepper, blur,
contrast, background, with the same keyword arguments, default ranges and per-image parameter
draws (np.random.seed(seed); the parameters are drawn with numpy in the reference's order, only
the per-pixel noise comes from the kernel's counter-based generator).  `zoom`, `resize` (cv2
cubic / area resampling) and `custom_transform` are not implemented and raise.
"""
from typing import Callable, Optional, Tuple

import numpy as np
import torch

from .. import ops

_NP = 16


class datatransform:
    """Sequence of augmentation operations applied to a CUDA batch (see module docstring)."""
    def __init__(self, n_channels: int = None, seed: Optional[int] = None, **kwargs) -> None:
        for k in ("zoom", "resize", "custom_transform"):
            if kwargs.get(k):
                raise NotImplementedError(
                    f"augmentation '{k}' is not implemented on the GPU path (cv2 resampling / "
                    "user callback); apply it to the data set up front")
        self.ch = n_channels
        self.rotation = kwargs.get('rotation')
        self.background = kwargs.get('background')
        rng = lambda v, d: d if v is True else v  # noqa: E731
        self.gauss = rng(kwargs.get('gauss_noise'), [0, 50])
        self.jitter = rng(kwargs.get('jitter'), [0, 50])
        self.poisson = rng(kwargs.get('poisson_noise'), [30, 40])
        self.salt_and_pepper = rng(kwargs.get('salt_and_pepper'), [0, 50])
        self.blur = rng(kwargs.get('blur'), [1, 50])
        self.contrast = rng(kwargs.get('contrast'), [5, 20])
        self.seed = seed
        if seed is not None:
            np.random.seed(seed)

    def run(self, images: torch.Tensor, targets: Optional[torch.Tensor] = None
            ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """images (n, h, w) CUDA fp32; targets (n, h, w) int64 label maps or None.  Returns the
        augmented images, min-max normalised to [0, 1] over the batch, and the (flipped) targets."""
        assert images.is_cuda and images.dim() == 3
        n, h, w = images.shape
        x = images.contiguous().float()
        P = np.zeros((n, _NP), np.float32)
        P[:, 0] = 9
        is_seq = lambda v: isinstance(v, (list, tuple))  # noqa: E731
        if self.rotation and targets is not None:
            for i in range(n):
                ft = np.random.randint(-1, 3)
                P[i, 0] = ft if (ft < 2 or h == w) else 9   # randint(-1, 3) never yields 3, as in the reference
        if is_seq(self.gauss):
            for i in range(n):
                P[i, 1] = 1e-4 * np.random.randint(self.gauss[0], self.gauss[1])
        row_shift = None
        if is_seq(self.jitter):
            from scipy import stats
            sh = np.zeros((n, h), np.int32)
            for i in range(n):
                amount = np.random.randint(self.jitter[0], self.jitter[1]) / 10
                sh[i] = stats.poisson.rvs(amount, loc=0, size=h)
            row_shift = torch.from_numpy(sh).to(x.device)
        if is_seq(self.poisson):
            for i in range(n):
                lam = np.random.randint(self.poisson[0], self.poisson[1])
                vals = int(torch.unique(x[i]).numel())
                P[i, 2] = (50 / lam) ** np.ceil(np.log2(max(vals, 1)))
        if is_seq(self.salt_and_pepper):
            for i in range(n):
                P[i, 3] = 1e-3 * np.random.randint(self.salt_and_pepper[0], self.salt_and_pepper[1])
        if is_seq(self.blur):
            for i in range(n):
                P[i, 4] = 5e-2 * np.random.randint(self.blur[0], self.blur[1])
        if is_seq(self.contrast):
            for i in range(n):
                P[i, 5] = np.random.randint(self.contrast[0], self.contrast[1]) / 10
        if self.background:
            for i in range(n):
                x0 = np.random.randint(0, h - h // 4)
                y0 = np.random.randint(0, w - w // 4)
                a, b = np.random.randint(10, 20, 2) / 10
                fwhm = np.random.randint(min([h, w]) // 4, min([h, w]) - min([h, w]) // 2)
                amp = 0.05 * np.random.randint(-10, 10)
                P[i, 6:11] = [amp, x0, y0, np.log(2) * a / fwhm ** 2, np.log(2) * b / fwhm ** 2]
        lo, hi = torch.aminmax(x)
        params = torch.from_numpy(P).to(x.device)
        y = torch.empty_like(x)
        scratch = torch.empty_like(x)
        lab_out = None
        if targets is not None:
            targets = targets.contiguous()
            assert targets.dtype == torch.int64 and targets.shape == x.shape
            lab_out = torch.empty_like(targets)
        minmax = torch.empty(2, device=x.device, dtype=torch.float32)
        seed = np.random.randint(0, 2 ** 31 - 1)
        ops.augment(x, y, scratch, targets, lab_out, params, row_shift, float(lo), float(hi), seed,
                    minmax)
        return y, lab_out


_AUG_KEYS = ["custom_transform", "zoom", "gauss_noise", "jitter", "poisson_noise", "contrast",
             "salt_and_pepper", "blur", "resize", "rotation", "background"]


def seg_augmentor(nb_classes: int, **kwargs) -> Optional[Callable]:
    """augment_fn(images (n,1,h,w), labels, seed) for BaseTrainer.data_augmentation, or None when
    no augmentation kwargs are given (atomai/transforms/imaug.py:406-432)."""
    augdict = {k: kwargs[k] for k in _AUG_KEYS if k in kwargs.keys()}
    if len(augdict) == 0:
        return None
    datatransform(nb_classes, None, **augdict)      # validate the kwargs now, not mid-training

    def augmentor(images, labels, seed):
        dev = "cuda"
        images = images.to(dev)
        labels = labels.to(dev)
        dt = datatransform(nb_classes, seed, **augdict)
        lab = labels[:, 0] if labels.dim() == 4 else labels
        out, lab_out = dt.run(images[:, 0], lab.long())
        out = out[:, None]
        if nb_classes == 1:
            lab_out = lab_out[:, None].float()
        return out, lab_out
    return augmentor


def imspec_augmentor(in_dim: Tuple[int], out_dim: Tuple[int], **kwargs) -> Optional[Callable]:
    """Image-side augmentation for im2spec models (atomai/transforms/imaug.py:435-457)."""
    keys = [k for k in _AUG_KEYS if k not in ("zoom", "resize", "rotation")]
    augdict = {k: kwargs[k] for k in keys if k in kwargs.keys()}
    if len(augdict) == 0:
        return None
    if len(in_dim) < len(out_dim):
        raise NotImplementedError("The built-in data augmentor works only" +
                                  " for img->spec models (i.e. input is image)")
    datatransform(None, None, **augdict)

    def augmentor(features, targets, seed):
        features = features.to("cuda")
        out, _ = datatransform(None, seed, **augdict).run(features[:, 0], None)
        return out[:, None], targets.to("cuda")
    return augmentor


def reg_augmentor(**kwargs) -> Optional[Callable]:
    """Image-only noise augmentation for Regressor / Classifier (atomai/transforms/imaug.py:461-478):
    gauss_noise, jitter, poisson_noise, contrast, salt_and_pepper, blur, background on the GPU,
    targets unchanged.  Other augmentation kwargs (custom_transform, zoom, resize, rotation) raise
    NotImplementedError."""
    for k in ("custom_transform", "zoom", "resize", "rotation"):
        if kwargs.get(k):
            raise NotImplementedError(
                f"augmentation '{k}' is not implemented for Regressor / Classifier on the GPU path")
    keys = ["gauss_noise", "jitter", "poisson_noise", "contrast", "salt_and_pepper", "blur",
            "background"]
    augdict = {k: kwargs[k] for k in keys if k in kwargs.keys()}
    if len(augdict) == 0:
        return None
    datatransform(None, None, **augdict)

    def augmentor(features, targets, seed):
        features = features.to("cuda")
        if features.shape[1] != 1:
            raise NotImplementedError("reg_augmentor augments single-channel images only")
        out, _ = datatransform(None, seed, **augdict).run(features[:, 0], None)
        return out[:, None], targets.to("cuda")
    return augmentor
