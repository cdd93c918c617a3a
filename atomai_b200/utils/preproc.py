"""
Data -> tensors/batches for the trainers: same function names, argument meaning and return
values as the reference's atomai/utils/preproc.py (:18-441, :798-825) for the functions the hot
path uses.  This is host-side plumbing (numpy/torch); the data-parallel sharder plugs in here
(`shard_batches`, SURVEY.md §8e).
"""
import warnings
from typing import List, Optional, Tuple, Type, Union

import numpy as np
import torch

Arr = Union[np.ndarray, torch.Tensor]


def num_classes_from_labels(labels: Arr) -> int:
    """Number of classes from masks: labels must be 0..K-1 without gaps; two label values mean
    one (binary) class (atomai/utils/preproc.py:18-41)."""
    vals = np.unique(labels.cpu().numpy() if isinstance(labels, torch.Tensor) else labels)
    if vals.min() != 0:
        raise AssertionError("Labels should start from 0")
    if np.any(np.diff(vals) != 1):
        raise AssertionError("Mask values should be in range between "
                             "0 and total number of classes "
                             "with an increment of 1")
    k = len(vals)
    return k - 1 if k == 2 else k


def _add_channel(a: Arr, what: str) -> Arr:
    warnings.warn(f'Adding a channel dimension of 1 to {what}', UserWarning)
    return a[:, None]


def check_image_dims(X_train, y_train, X_test, y_test, num_classes: int):
    """Adds the pseudo channel dimension where missing (preproc.py:43-74)."""
    if X_train.ndim == 3:
        X_train = _add_channel(X_train, "training images")
    if X_test.ndim == 3:
        X_test = _add_channel(X_test, "test images")
    if num_classes == 1 and y_train.ndim == 3:
        y_train = _add_channel(y_train, "training labels")
    if num_classes == 1 and y_test.ndim == 3:
        y_test = _add_channel(y_test, "test labels")
    return X_train, y_train, X_test, y_test


def check_signal_dims(X_train, y_train, X_test, y_test):
    """Channel dims for im2spec / spec2im data (preproc.py:77-135)."""
    if X_train.ndim > y_train.ndim:            # images -> spectra
        img_nd, sig_nd = 3, 2
        if X_train.ndim == img_nd:
            X_train = _add_channel(X_train, "training images")
        if X_test.ndim == img_nd:
            X_test = _add_channel(X_test, "test images")
        if y_train.ndim == sig_nd:
            y_train = _add_channel(y_train, "training spectra")
        if y_test.ndim == sig_nd:
            y_test = _add_channel(y_test, "test spectra")
    elif X_train.ndim < y_train.ndim:          # spectra -> images
        if X_train.ndim == 2:
            X_train = _add_channel(X_train, "training images")
        if X_test.ndim == 2:
            X_test = _add_channel(X_test, "test images")
        if y_train.ndim == 3:
            y_train = _add_channel(y_train, "training spectra")
        if y_test.ndim == 3:
            y_test = _add_channel(y_test, "test spectra")
        if X_train.shape[1:] != X_test.shape[1:] or y_train.shape[1:] != y_test.shape[1:]:
            raise ValueError("The image/spectra dimensions must be" +
                             " the same for training and test data")
    return X_train, y_train, X_test, y_test


def get_array_memsize(X_arr: Optional[Arr], precision: str = "single") -> float:
    """Bytes the array takes once cast to single/double precision (preproc.py:138-167)."""
    if X_arr is None:
        return 0
    if isinstance(X_arr, torch.Tensor):
        nbytes, wide = X_arr.numel() * X_arr.element_size(), X_arr.element_size() == 8
        known = X_arr.dtype in (torch.float32, torch.float64, torch.int32, torch.int64)
    else:
        nbytes, wide = X_arr.nbytes, X_arr.dtype.itemsize == 8
        known = X_arr.dtype in (np.float32, np.float64, np.int32, np.int64)
    if precision not in ("single", "double"):
        raise NotImplementedError("Specify 'single' or 'double' precision type")
    if not known:
        warnings.warn("Data type is not understood", UserWarning)
        return nbytes
    if precision == "single":
        return nbytes / 2 if wide else nbytes
    return nbytes if wide else nbytes * 2


def array2list_(x: Arr, batch_size: int, store_on_cpu: bool = False):
    if not isinstance(x, (np.ndarray, torch.Tensor)):
        raise TypeError("Provide data as numpy array or torch tensor")
    if isinstance(x, torch.Tensor):
        x = x.to('cuda' if torch.cuda.is_available() and not store_on_cpu else 'cpu')
        if store_on_cpu and torch.cuda.is_available() and not x.is_pinned():
            x = x.pin_memory()       # host-resident batches are copied asynchronously each step
    n_batches = x.shape[0] // batch_size
    x = x[:n_batches * batch_size]
    return np.split(x, n_batches) if isinstance(x, np.ndarray) else torch.chunk(x, n_batches)


def array2list(X_train, y_train, X_test, y_test, batch_size: int, memory_alloc: float = 4):
    """Lists of batch-sized chunks, resident on the GPU when they fit `memory_alloc` GB
    (preproc.py:170-201); remainders are dropped."""
    total = sum(get_array_memsize(x) for x in (X_train, y_train, X_test, y_test))
    on_cpu = (total / 1e9) > memory_alloc
    return tuple(array2list_(x, batch_size, on_cpu) for x in (X_train, y_train, X_test, y_test))


def preprocess_training_image_data_(images_all, labels_all, images_test_all, labels_test_all):
    """Type/dim checks and dtype casts for segmentation data (preproc.py:204-234)."""
    data = (images_all, labels_all, images_test_all, labels_test_all)
    all_np = all(isinstance(i, np.ndarray) for i in data)
    all_t = all(isinstance(i, torch.Tensor) for i in data)
    if not all_np and not all_t:
        raise TypeError("Provide training and test data in the form" +
                        " of numpy arrays or torch tensors")
    num_classes = num_classes_from_labels(labels_all)
    X, y, Xt, yt = check_image_dims(*data, num_classes)
    if all_np:
        X, y, Xt, yt = (torch.from_numpy(np.ascontiguousarray(a)) for a in (X, y, Xt, yt))
    X, Xt = X.float(), Xt.float()
    if num_classes > 1:
        y, yt = y.long(), yt.long()
    else:
        y, yt = y.float(), yt.float()
    return X, y, Xt, yt, num_classes


def preprocess_training_image_data(images_all, labels_all, images_test_all, labels_test_all,
                                   batch_size: int, memory_alloc: float = 4):
    """(train image batches, train label batches, test ..., nb_classes) — preproc.py:237-278."""
    *tensors, num_classes = preprocess_training_image_data_(
        images_all, labels_all, images_test_all, labels_test_all)
    return (*array2list(*tensors, batch_size, memory_alloc), num_classes)


def preprocess_training_imspec_data_(X_train, y_train, X_test, y_test):
    """Checks + float casts for im2spec/spec2im data; returns dims (preproc.py:281-313)."""
    data = (X_train, y_train, X_test, y_test)
    all_np = all(isinstance(i, np.ndarray) for i in data)
    all_t = all(isinstance(i, torch.Tensor) for i in data)
    if not all_np and not all_t:
        raise TypeError("Provide training and test data in the form" +
                        " of numpy arrays or torch tensors")
    X_train, y_train, X_test, y_test = check_signal_dims(*data)
    in_dim, out_dim = tuple(X_train.shape[2:]), tuple(y_train.shape[2:])
    if all_np:
        X_train, y_train, X_test, y_test = (torch.from_numpy(np.ascontiguousarray(a))
                                            for a in (X_train, y_train, X_test, y_test))
    X_train, y_train, X_test, y_test = (a.float() for a in (X_train, y_train, X_test, y_test))
    return X_train, y_train, X_test, y_test, (in_dim, out_dim)


def preprocess_training_imspec_data(X_train, y_train, X_test, y_test, batch_size: int,
                                    memory_alloc: float = 4):
    *tensors, dims = preprocess_training_imspec_data_(X_train, y_train, X_test, y_test)
    return (*array2list(*tensors, batch_size, memory_alloc), dims)


def preprocess_denoiser_data(X_train, y_train, X_test, y_test):
    """Noisy / clean image pairs -> float32 (n, 1, h, w) tensors (preproc.py:698-758): a
    channel dimension is added to 3-D inputs with a UserWarning; mixed numpy / torch inputs raise
    TypeError, noisy / clean shape mismatches ValueError."""
    data = (X_train, y_train, X_test, y_test)
    all_np = all(isinstance(i, np.ndarray) for i in data)
    all_t = all(isinstance(i, torch.Tensor) for i in data)
    if not all_np and not all_t:
        raise TypeError(
            "Provide training and test data in the form of numpy arrays or torch tensors")
    what = ("noisy training images", "clean training images", "noisy test images",
            "clean test images")
    out = []
    for a, w in zip(data, what):
        if a.ndim == 3:
            warnings.warn(f"Adding channel dimension of 1 to {w}", UserWarning)
            a = a[:, None]
        out.append(torch.from_numpy(np.ascontiguousarray(a)).float() if all_np else a.float())
    X_train, y_train, X_test, y_test = out
    if X_train.shape != y_train.shape:
        raise ValueError("Noisy and clean training images must have the same shape")
    if X_test.shape != y_test.shape:
        raise ValueError("Noisy and clean test images must have the same shape")
    return X_train, y_train, X_test, y_test


def _check_numpy_or_torch(data) -> bool:
    all_np = all(isinstance(i, np.ndarray) for i in data)
    all_t = all(isinstance(i, torch.Tensor) for i in data)
    if not all_np and not all_t:
        raise TypeError(
            "Provide training and test data in the form of numpy arrays or torch tensors")
    return all_np


def _image_channel(X_train, X_test):
    if X_train.ndim == 3:
        warnings.warn('Adding a channel dimension of 1 to training images', UserWarning)
        X_train = X_train[:, None]
    if X_test.ndim == 3:
        warnings.warn('Adding a channel dimension of 1 to test images', UserWarning)
        X_test = X_test[:, None]
    return X_train, X_test


def preprocess_training_reg_data_(X_train, y_train, X_test, y_test):
    """Images (n, c, h, w) or (n, h, w) and targets (n, out_dim) or (n,) -> float32 tensors; the
    missing channel / target dimension is added with a UserWarning (preproc.py:481-528)."""
    all_np = _check_numpy_or_torch((X_train, y_train, X_test, y_test))
    X_train, X_test = _image_channel(X_train, X_test)
    if y_train.ndim == 1:
        warnings.warn('Adding a channel dimension of 1 to training targets', UserWarning)
        y_train = y_train[:, None]
    if y_test.ndim == 1:
        warnings.warn('Adding a channel dimension of 1 to test targets', UserWarning)
        y_test = y_test[:, None]
    tor = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).float()) if all_np \
        else (lambda a: a.float())
    return tor(X_train), tor(y_train), tor(X_test), tor(y_test)


def preprocess_training_reg_data(X_train, y_train, X_test, y_test, batch_size: int,
                                 memory_alloc: float = 4):
    """preprocess_training_reg_data_ + lists of batches (preproc.py:531-571)."""
    return array2list(*preprocess_training_reg_data_(X_train, y_train, X_test, y_test),
                      batch_size, memory_alloc)


def preprocess_training_cls_data_(X_train, y_train, X_test, y_test):
    """Images (n, c, h, w) or (n, h, w) -> float32, labels must be 1-D int64 (TypeError otherwise;
    preproc.py:613-656)."""
    all_np = _check_numpy_or_torch((X_train, y_train, X_test, y_test))
    X_train, X_test = _image_channel(X_train, X_test)
    if y_train.dtype not in (torch.int64, np.int64):
        raise TypeError(
            "Provide training labels as 1D array of integers (numpy.int64 or torch.int64)")
    if y_test.dtype not in (torch.int64, np.int64):
        raise TypeError(
            "Provide test labels as 1D array of integers (numpy.int64 or torch.int64)")
    if all_np:
        return (torch.from_numpy(np.ascontiguousarray(X_train)).float(),
                torch.from_numpy(np.ascontiguousarray(y_train)),
                torch.from_numpy(np.ascontiguousarray(X_test)).float(),
                torch.from_numpy(np.ascontiguousarray(y_test)))
    return X_train.float(), y_train, X_test.float(), y_test


def preprocess_training_cls_data(X_train, y_train, X_test, y_test, batch_size: int,
                                 memory_alloc: float = 4):
    """preprocess_training_cls_data_ + lists of batches (preproc.py:659-695)."""
    return array2list(*preprocess_training_cls_data_(X_train, y_train, X_test, y_test),
                      batch_size, memory_alloc)


def init_dataloaders(X_train, y_train, X_test, y_test, batch_size: int, memory_alloc: float = 4):
    """Train (shuffled) / test DataLoaders over device-resident TensorDatasets, drop_last=True
    (preproc.py:365-388)."""
    dev = 'cuda' if torch.cuda.is_available() else 'cpu'
    if sum(get_array_memsize(x) for x in (X_train, y_train, X_test, y_test)) / 1e9 > memory_alloc:
        dev = 'cpu'
    X_train, y_train, X_test, y_test = (t.to(dev) for t in (X_train, y_train, X_test, y_test))
    ds = torch.utils.data.TensorDataset
    train_loader = torch.utils.data.DataLoader(ds(X_train, y_train), batch_size=batch_size,
                                               shuffle=True, drop_last=True)
    test_loader = torch.utils.data.DataLoader(ds(X_test, y_test), batch_size=batch_size,
                                              drop_last=True)
    return train_loader, test_loader


def init_dataloader(X, shuffle: bool = True, **kwargs: int):
    batch_size = kwargs.get("batch_size", len(X))
    X = (X,) if isinstance(X, torch.Tensor) else X
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(*X),
                                       batch_size=batch_size, shuffle=shuffle)


def init_fcnn_dataloaders(X_train, y_train, X_test, y_test, batch_size: int,
                          num_classes: Optional[int] = None, memory_alloc: float = 4):
    *tensors, num_classes = preprocess_training_image_data_(X_train, y_train, X_test, y_test)
    train_loader, test_loader = init_dataloaders(*tensors, batch_size, memory_alloc)
    return train_loader, test_loader, num_classes


def init_imspec_dataloaders(X_train, y_train, X_test, y_test, batch_size: int,
                            memory_alloc: float = 4):
    *tensors, dims = preprocess_training_imspec_data_(X_train, y_train, X_test, y_test)
    train_loader, test_loader = init_dataloaders(*tensors, batch_size, memory_alloc)
    return train_loader, test_loader, dims


def torch_format_image(image_data: np.ndarray, norm: bool = True) -> torch.Tensor:
    """(n,h,w) or (n,1,h,w) -> float32 (n,1,h,w) tensor, globally min-max normalised in float64
    exactly like the reference (preproc.py:798-825) so predictions see identical inputs."""
    if image_data.ndim not in [3, 4]:
        raise AssertionError("Provide image(s) as 3D (n, h, w) or 4D (n, 1, h, w) tensor")
    if image_data.ndim == 3:
        image_data = np.expand_dims(image_data, axis=1)
    if norm:
        image_data = (image_data - image_data.min()) / np.ptp(image_data)
    return torch.from_numpy(image_data).float()


def torch_format_spectra(spectra: np.ndarray, norm: bool = False) -> torch.Tensor:
    if spectra.ndim not in [2, 3]:
        raise AssertionError("Provide spectra as 2D (n, length) or 3D (n, 1, length) tensor")
    if spectra.ndim == 2:
        spectra = np.expand_dims(spectra, axis=1)
    if norm:
        spectra = (spectra - spectra.min()) / np.ptp(spectra)
    return torch.from_numpy(spectra).float()


def shard_batches(batches: List[torch.Tensor], rank: int, world: int) -> List[torch.Tensor]:
    """Data-parallel sharding (new; the reference is single-device): rank r keeps rows
    [r*B/G, (r+1)*B/G) of every mini-batch so that the union over ranks is the reference's batch."""
    if world == 1:
        return list(batches)
    out = []
    for b in batches:
        n = b.shape[0]
        assert n % world == 0, f"batch of {n} does not divide over {world} ranks"
        k = n // world
        out.append(b[rank * k:(rank + 1) * k].contiguous())
    return out


def create_batches(array, batch_size: int) -> list:
    """Consecutive slices of `batch_size` rows of an array / tensor, the last one possibly shorter
    (atomai/utils/preproc.py:932-935)."""
    nb = -(-array.shape[0] // batch_size)
    return [array[k * batch_size:(k + 1) * batch_size] for k in range(nb)]


def prepare_gp_input(sparse_image: np.ndarray):
    """GP inputs of a sparse scan whose unmeasured pixels are zero (atomai/utils/preproc.py:938-947):
    the indices (N, ndim) of the non-zero pixels in row-major order, their values (N,), and the
    indices of every pixel (H*W..., ndim).  The full grid is numpy's meshgrid (default 'xy'
    indexing) stacked and transposed, whose rows for a 2-D image run in row-major order, so a
    prediction over it reshapes back into the image."""
    measured = np.nonzero(sparse_image)
    x_train = np.stack(measured, axis=1)
    y_train = sparse_image[measured]
    axes = [np.arange(n) for n in sparse_image.shape]
    x_full = np.array(np.meshgrid(*axes)).T.reshape(-1, sparse_image.ndim)
    return x_train, y_train, x_full
