"""
Image helpers on the prediction path (host-side numpy): padding to the network's downsampling
factor, binary thresholding and resizing — atomai/utils/img.py:20-40, 112-135, 554-564; sub-image
extraction around atoms, and the random patches and patch / spectrum pairs that make training
sets (atomai/utils/img.py:138-452), whose crops are gathers on the GPU; the blob-size filter of
segmented frames (atomai/utils/img.py:567-625), labelled on the GPU; the FFT-subtraction defect
map (atomai/utils/img.py:455-499), whose 2-D transforms run on the GPU in float64.
"""
from numbers import Integral, Real
from typing import List, Tuple, Union

import numpy as np


def img_pad(image_data: np.ndarray, pooling: int) -> np.ndarray:
    """Zero-pads (n, h, w) at the bottom/right so that h and w are divisible by `pooling`
    (atomai/utils/img.py:112-135; float64 result like the reference's np.concatenate)."""
    pooling = int(pooling)
    n, h, w = image_data.shape
    ph, pw = (-h) % pooling, (-w) % pooling
    if ph == 0 and pw == 0:
        return image_data
    out = np.zeros((n, h + ph, w + pw), dtype=np.result_type(image_data.dtype, np.float64))
    out[:, :h, :w] = image_data
    return out


def cv_thresh(imgdata: np.ndarray, threshold: float = .5) -> np.ndarray:
    """cv2.threshold(img, threshold, 1, THRESH_BINARY): 1.0 where img > threshold else 0.0, same
    dtype as the input (atomai/utils/img.py:554-564).  Pure numpy so cv2 is not a dependency."""
    return (imgdata > threshold).astype(imgdata.dtype)


# ------------------------------------------------------------------ blob filtering
# atomai/utils/img.py:567-625 runs cv2.threshold, scipy.ndimage.label (4-connectivity) and
# ndimage.sum frame by frame.  Here the threshold, the labelling and the size test of every frame
# of a stack run in csrc/blobs.cu; the host only checks the arguments.
_BLOB_NP = tuple(np.dtype(t) for t in (np.uint8, np.int16, np.uint16, np.float32, np.float64))


def _blob_check(imgdata, ndim: int, im_thresh, blob_thresh, filter_) -> bool:
    """the argument checks of filter_cells[_], all before any device work; returns `above`"""
    import torch
    if _is_cuda(imgdata):
        ok = imgdata.dtype in (torch.uint8, torch.int16, torch.uint16, torch.float32, torch.float64)
    elif isinstance(imgdata, np.ndarray):
        ok = imgdata.dtype in _BLOB_NP
    else:
        raise TypeError(f"imgdata must be a numpy array or a CUDA tensor, not {type(imgdata)}")
    if imgdata.ndim != ndim:
        raise ValueError(f"imgdata must be {ndim}-D, got shape {tuple(imgdata.shape)}")
    if not ok:
        raise TypeError(f"dtype {imgdata.dtype} is not supported: cv2.threshold takes uint8, int16, "
                        "uint16, float32 and float64")
    for name, v in (("im_thresh", im_thresh), ("blob_thresh", blob_thresh)):
        if not isinstance(v, Real):
            raise TypeError(f"{name} must be a real number, not {type(v)}")
    if not np.isfinite(float(im_thresh)):
        raise ValueError(f"im_thresh must be finite, got {im_thresh}")
    h, w = imgdata.shape[-2:]
    if h * w >= 2**31:
        raise ValueError(f"frames of {h} x {w} pixels are too large: at most 2^31 - 1 pixels")
    if (ndim == 2 or imgdata.shape[0]) and not h * w:
        raise TypeError("cv2.threshold returns no image for an empty frame")
    return bool(filter_ == 'above')


def _filter_blobs(stack, im_thresh, blob_thresh, above: bool, out_dtype):
    """the kept-blob mask of every frame of an (n, h, w) stack, numpy or CUDA like the stack"""
    import torch
    from .. import ops
    from .graphx import _check_free
    cuda = _is_cuda(stack)
    if 0 in tuple(stack.shape):
        if cuda:
            return torch.zeros(stack.shape, dtype=out_dtype, device=stack.device)
        return np.zeros(stack.shape, out_dtype)
    if not cuda:
        out_dtype = torch.from_numpy(np.zeros(0, out_dtype)).dtype
    npix = int(np.prod(stack.shape, dtype=np.int64))
    in_bytes = stack.element_size() if cuda else stack.itemsize
    out_bytes = torch.empty((), dtype=out_dtype).element_size()
    _check_free(npix * (8 + out_bytes + (0 if cuda else in_bytes)), "the blob filter")
    if cuda:
        img = stack.contiguous()
    else:
        if not torch.cuda.is_available():
            raise RuntimeError("this function runs on a CUDA device; none is available")
        img = torch.from_numpy(np.ascontiguousarray(stack)).to("cuda")
    labels = torch.empty(img.shape, dtype=torch.int32, device=img.device)
    counts = torch.empty_like(labels)
    out = torch.empty(img.shape, dtype=out_dtype, device=img.device)
    ops.blob_filter(img, float(im_thresh), float(blob_thresh), above, labels, counts, out)
    return out if cuda else out.cpu().numpy()


def filter_cells_(imgdata: np.ndarray,
                  im_thresh: float = .5,
                  blob_thresh: int = 150,
                  filter_: str = 'below') -> np.ndarray:
    """Removes the blobs of one (h, w) frame that are smaller than `blob_thresh` pixels (or, with
    filter_='above', larger), after thresholding at `im_thresh` (atomai/utils/img.py:567-584).
    Blobs are 4-connected; the result is an int32 0/1 (h, w) array, or a CUDA tensor for a CUDA
    input.  Input dtypes are cv2.threshold's: uint8, int16, uint16, float32 and float64."""
    import torch
    above = _blob_check(imgdata, 2, im_thresh, blob_thresh, filter_)
    out = _filter_blobs(imgdata[None], im_thresh, blob_thresh, above,
                        torch.int32 if _is_cuda(imgdata) else np.int32)
    return out[0]


def filter_cells(imgdata: np.ndarray,
                 im_thresh: float = 0.5,
                 blob_thresh: int = 50,
                 filter_: str = 'below') -> np.ndarray:
    """filter_cells_ on every frame of an (n, h, w) stack (atomai/utils/img.py:598-625); the
    result has the input's shape and dtype, 1 on the kept blobs.  All frames run in one pass of
    each GPU kernel."""
    above = _blob_check(imgdata, 3, im_thresh, blob_thresh, filter_)
    return _filter_blobs(imgdata, im_thresh, blob_thresh, above, imgdata.dtype)


# ------------------------------------------------------------------ FFT subtraction
# atomai/utils/img.py:455-499 runs scipy.fftpack.fft2 / ifft2 on the host.  Here the transforms,
# the shifts, the disk mask and the normalisation run in csrc/fft.cu, always in float64; a
# complex64 or float32 result is rounded once, at the store.  The host only checks the arguments
# and works out the mask's box from the reference's numpy slices.
_FFT_NP = tuple(np.dtype(t) for t in (
    np.bool_, np.uint8, np.int8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64,
    np.float16, np.float32, np.float64, np.complex64, np.complex128))
_FFT_SINGLE = tuple(np.dtype(t) for t in (np.float16, np.float32, np.complex64))


def _fft_dtype(a) -> np.dtype:
    """the numpy dtype of a numpy array or CUDA tensor the FFT kernels load; TypeError otherwise"""
    import torch
    if _is_cuda(a):
        from .. import ops
        if a.dtype not in ops.FFT_CODES:
            raise TypeError(f"dtype {a.dtype} is not supported by the GPU FFT")
        return np.dtype(str(a.dtype).replace("torch.", "").replace("bool", "bool_"))
    if isinstance(a, torch.Tensor) or not isinstance(a, np.ndarray):
        raise TypeError(f"expected a numpy array or a CUDA tensor, not {type(a)}")
    if a.dtype not in _FFT_NP:
        raise TypeError(f"dtype {a.dtype} is not supported by the GPU FFT: it takes bool, integers "
                        "of up to 64 bits, float16/32/64 and complex64/128")
    return a.dtype


def _fft_shape(shape) -> Tuple[int, int]:
    """(h, w) of a 2-D image within the transform's size limits; ValueError otherwise"""
    from .. import _C
    if len(shape) != 2:
        raise ValueError(f"the image must be 2-D, got shape {tuple(shape)}")
    for n in shape:
        if n < 1:
            raise ValueError(f"invalid number of data points ({list(shape)}) specified")
        if n > _C.FFT_MAX_SIDE and (n & (n - 1) or n > _C.FFT_MAX_POW2):
            raise ValueError(f"a side of {n} is too long for the GPU FFT: at most "
                             f"{_C.FFT_MAX_SIDE}, or a power of two up to {_C.FFT_MAX_POW2}")
    return int(shape[0]), int(shape[1])


def _mask_box(shape, maskratio) -> Tuple[int, int, int]:
    """(r0, c0, l) of the disk atomai/utils/img.py:467-471 zeroes: F3[m-l:m+l, m-l:m+l] times
    (1 - mask) of the (2l, 2l) disk, both from shape[0].  The same expressions raise the same
    errors (ZeroDivisionError for maskratio=0); slices that do not broadcast with the mask raise
    ValueError, as numpy does; l = 0 when nothing is masked."""
    l = int(shape[0] / maskratio)
    m = int(shape[0] / 2)
    rows, cols = range(shape[0])[m - l:m + l], range(shape[1])[m - l:m + l]
    box, mask = (len(rows), len(cols)), (max(2 * l, 0),) * 2
    try:
        ok = np.broadcast_shapes(np.broadcast_shapes(box, mask), box) == box
    except ValueError:
        ok = False
    if not ok:
        raise ValueError(f"the mask of shape {mask} does not broadcast into the slice of shape "
                         f"{box} (image {tuple(shape)}, maskratio {maskratio})")
    return (rows.start, cols.start, l) if l > 0 and box == mask else (0, 0, 0)


def _to_device(a):
    import torch
    if _is_cuda(a):
        return a.contiguous()
    if not torch.cuda.is_available():
        raise RuntimeError("this function runs on a CUDA device; none is available")
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda")


def _torch_dtype(dt: np.dtype):
    import torch
    return torch.from_numpy(np.zeros(0, dt)).dtype


def FFTmask(imgsrc: np.ndarray, maskratio: int = 10) -> Tuple[np.ndarray]:
    """Returns F2, the centred 2-D FFT of an (h, w) image, and F3, a copy of F2 with a disk of
    radius shape[0] / maskratio zeroed around the centre (atomai/utils/img.py:455-472).  The
    transform runs on the GPU in float64; F2 and F3 are complex64 for float16, float32 and
    complex64 input and complex128 otherwise, numpy arrays for numpy input and CUDA tensors for
    CUDA input.  Each side may be up to 4096 long, or a power of two up to 8192."""
    import torch
    from .. import ops
    from .graphx import _check_free
    dt = _fft_dtype(imgsrc)
    h, w = _fft_shape(imgsrc.shape)
    r0, c0, l = _mask_box(imgsrc.shape, maskratio)
    out_dt = np.dtype(np.complex64 if dt in _FFT_SINGLE else np.complex128)
    _check_free(h * w * (2 * out_dt.itemsize + (0 if _is_cuda(imgsrc) else dt.itemsize))
                + ops.fft2_workspace_bytes(h, w), "FFTmask")
    img = _to_device(imgsrc)
    f2 = torch.empty((h, w), dtype=_torch_dtype(out_dt), device=img.device)
    f3 = torch.empty_like(f2)
    ops.fft2_mask(img, r0, c0, l, f2, f3)
    if _is_cuda(imgsrc):
        return f2, f3
    return f2.cpu().numpy(), f3.cpu().numpy()


def FFTsub(imgsrc: np.ndarray, imgfft: np.ndarray) -> np.ndarray:
    """Reconstructs an image from the filtered, centred spectrum `imgfft` (complex64 or
    complex128), subtracts it from `imgsrc` and min-max normalises the absolute difference
    (atomai/utils/img.py:475-486); a constant difference gives NaN, like the reference's 0 / 0.
    Both must be 2-D of the same shape.  The result's dtype is the reference's, the real dtype of
    np.result_type(imgsrc, the spectrum's real dtype), computed in float64 on the GPU; it is a
    numpy array or a CUDA tensor like `imgsrc`."""
    import torch
    from .. import ops
    from .graphx import _check_free
    src_dt, fft_dt = _fft_dtype(imgsrc), _fft_dtype(imgfft)
    if fft_dt.kind != "c":
        raise TypeError(f"imgfft must be a complex64 or complex128 spectrum, not {fft_dt}")
    h, w = _fft_shape(imgsrc.shape)
    if tuple(imgfft.shape) != (h, w):
        raise ValueError(f"imgsrc {tuple(imgsrc.shape)} and imgfft {tuple(imgfft.shape)} must "
                         "have the same 2-D shape")
    out_dt = np.result_type(src_dt, np.empty(0, fft_dt).real.dtype)
    out_dt = np.empty(0, out_dt).real.dtype
    _check_free(h * w * (out_dt.itemsize + (0 if _is_cuda(imgsrc) else src_dt.itemsize)
                         + (0 if _is_cuda(imgfft) else fft_dt.itemsize))
                + ops.fft2_workspace_bytes(h, w), "FFTsub")
    src = _to_device(imgsrc)
    spec = _to_device(imgfft).to(src.device)
    out = torch.empty((h, w), dtype=_torch_dtype(out_dt), device=src.device)
    ops.fft2_sub(src, spec, out)
    return out if _is_cuda(imgsrc) else out.cpu().numpy()


def threshImg(diff: np.ndarray,
              threshL: float = 0.25,
              threshH: float = 0.75) -> np.ndarray:
    """Marks the pixels of `diff` below threshL or above threshH as defects
    (atomai/utils/img.py:489-499): a bool array, or a bool tensor for a tensor input."""
    import torch
    if isinstance(diff, torch.Tensor):
        return torch.logical_or(diff < threshL, diff > threshH)
    return (diff < threshL) + (diff > threshH)


def img_resize(image_data: np.ndarray, rs: Tuple[int], round_: bool = False) -> np.ndarray:
    """Resizes a stack of images (atomai/utils/img.py:20-40); needs cv2 like the reference."""
    import cv2
    if rs[0] != rs[1]:
        rs = (rs[1], rs[0])
    if image_data.shape[1:3] == rs:
        return image_data.copy()
    out = np.zeros((image_data.shape[0], rs[0], rs[1]))
    inter = cv2.INTER_AREA if image_data.shape[1] > rs[0] else cv2.INTER_CUBIC
    for i, img in enumerate(image_data):
        img = cv2.resize(img, (rs[0], rs[1]), interpolation=inter)
        out[i] = np.round(img) if round_ else img
    return out


# ------------------------------------------------------------------ sub-image extraction
# SURVEY.md §8(f) rank 2: the step between Segmentor.predict and the VAE path
# (atomai/utils/img.py:138-180, 183-350, 502-551).  The reference crops window by window in a
# Python loop; here every window of an image is one vectorised gather.  Semantics that tests
# pin against the reference: np.around (half-to-even) centre rounding, windows that do not fit
# are dropped, so are windows containing NaN, numpy's negative-index wrap-around is honoured
# (a window whose start AND stop are negative is a legal crop from the far edge), coordinates
# are returned un-rounded, empty results are (None, None) / three empty lists.
def _window_starts(centres: np.ndarray, r: int, dim: int):
    """start index of each window along one axis (after numpy's negative-index rules) and a mask
    of the windows whose slice has exactly r elements."""
    half = r // 2
    start = centres - half
    stop = centres + half + (1 if r % 2 else 0)
    ok = (start >= 0) & (stop <= dim)
    wrap = (stop < 0) & (start + dim >= 0)          # both negative: slice counted from the end
    start = np.where(wrap, start + dim, start)
    return start, ok | wrap


def get_imgstack(imgdata: np.ndarray, coord: np.ndarray, r: int):
    """Sub-images of side `r` centred at the (x, y) coordinates of ONE image (h, w[, c]);
    returns (stack, kept coordinates) or (None, None) — atomai/utils/img.py:138-180."""
    coord = np.asarray(coord)
    if len(coord) == 0:
        return None, None
    r = int(r)
    cx = np.around(coord[:, 0]).astype(np.int64)
    cy = np.around(coord[:, 1]).astype(np.int64)
    sx, okx = _window_starts(cx, r, imgdata.shape[0])
    sy, oky = _window_starts(cy, r, imgdata.shape[1])
    keep = okx & oky
    if not keep.any():
        return None, None
    idx = np.nonzero(keep)[0]
    ar = np.arange(r)
    rows = (sx[idx, None] + ar[None, :])[:, :, None]            # (k, r, 1)
    cols = (sy[idx, None] + ar[None, :])[:, None, :]            # (k, 1, r)
    stack = imgdata[rows, cols]                                 # (k, r, r[, c]) — one gather
    if np.issubdtype(stack.dtype, np.floating):
        finite = ~np.isnan(stack.reshape(len(idx), -1)).any(1)
        if not finite.any():
            return None, None
        stack, idx = stack[finite], idx[finite]
    return np.ascontiguousarray(stack), coord[idx]


def extract_subimages_cuda(imgdata, coordinates, window_size: int, coord_class: int = 0):
    """extract_subimages for a CUDA image stack (n, h, w, c) fp32: the window bookkeeping (centre
    rounding, which windows fit, numpy's negative-index wrap) is the same host code as the numpy
    path, the crops themselves are ONE gather kernel over all frames
    (atomai_b200_gather_windows) that also flags windows containing NaN.  Returns
    (CUDA tensor (K, r, r, c), centres (K, 2) numpy, frame index (K,) numpy), or three empty
    lists when nothing fits (like the reference)."""
    import torch
    from .. import ops
    assert imgdata.is_cuda and imgdata.dim() == 4 and imgdata.dtype == torch.float32
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: np.concatenate((coordinates, np.zeros((coordinates.shape[0], 1))), axis=-1)}
    n, h, w, c = imgdata.shape
    r = int(window_size)
    rows, coms, frames = [], [], []
    for i, coord in zip(range(n), coordinates.values()):
        coord_i = np.asarray(coord)
        coord_i = coord_i[coord_i[:, 2] == coord_class][:, :2]
        if len(coord_i) == 0:
            continue
        cx = np.around(coord_i[:, 0]).astype(np.int64)
        cy = np.around(coord_i[:, 1]).astype(np.int64)
        sx, okx = _window_starts(cx, r, h)
        sy, oky = _window_starts(cy, r, w)
        idx = np.nonzero(okx & oky)[0]
        if len(idx) == 0:
            continue
        rows.append(np.stack([np.full(len(idx), i), sx[idx], sy[idx]], 1))
        coms.append(coord_i[idx])
        frames.append(np.ones(len(idx), int) * i)
    if not rows:
        return [], [], []
    table = torch.from_numpy(np.concatenate(rows).astype(np.int32)).to(imgdata.device)
    K = table.shape[0]
    out = torch.empty((K, r, r, c), device=imgdata.device, dtype=torch.float32)
    nanflag = torch.zeros(K, device=imgdata.device, dtype=torch.int32)
    ops.gather_windows(imgdata.contiguous(), table, r, out, nanflag)
    keep = (nanflag == 0).cpu().numpy()
    coms, frames = np.concatenate(coms), np.concatenate(frames)
    if not keep.all():
        if not keep.any():
            return [], [], []
        out = out[torch.from_numpy(keep).to(out.device)]
        coms, frames = coms[keep], frames[keep]
    return out, coms, frames


def extract_subimages(imgdata: np.ndarray, coordinates, window_size: int, coord_class: int = 0):
    """(sub-images, centres, frame index) around the atoms of class `coord_class` in a stack
    (n, h, w, c) with Locator-style coordinates {i: (N, 3)} — atomai/utils/img.py:298-350.
    Images are paired with the dictionary's VALUES in insertion order, like the reference.
    A CUDA tensor stack takes the gather-kernel path (extract_subimages_cuda)."""
    if hasattr(imgdata, "is_cuda") and imgdata.is_cuda:
        if imgdata.dim() == 2:
            imgdata = imgdata[None, ..., None]
        return extract_subimages_cuda(imgdata, coordinates, window_size, coord_class)
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: np.concatenate((coordinates, np.zeros((coordinates.shape[0], 1))), axis=-1)}
    if np.ndim(imgdata) == 2:
        imgdata = imgdata[None, ..., None]
    subimages_all, com_all, frames_all = [], [], []
    for i, (img, coord) in enumerate(zip(imgdata, coordinates.values())):
        coord_i = coord[coord[:, 2] == coord_class][:, :2]
        stack_i, com_i = get_imgstack(img, coord_i, window_size)
        if stack_i is None:
            continue
        subimages_all.append(stack_i)
        com_all.append(com_i)
        frames_all.append(np.ones(len(com_i), int) * i)
    if len(subimages_all) > 0:
        subimages_all = np.concatenate(subimages_all, axis=0)
        com_all = np.concatenate(com_all, axis=0)
        frames_all = np.concatenate(frames_all, axis=0)
    return subimages_all, com_all, frames_all


def imcrop_randpx(img: np.ndarray, window_size: int, num_images: int, random_state: int = 0):
    """`num_images` windows at distinct random pixels (np.random global state, same draw order as
    atomai/utils/img.py:183-211; `random_state` is accepted and ignored there too)."""
    seen, com = set(), []
    lo = window_size // 2 + 1
    while len(com) < num_images:
        x = np.random.randint(lo, img.shape[0] - window_size // 2 - 1)
        y = np.random.randint(lo, img.shape[1] - window_size // 2 - 1)
        if (x, y) not in seen:
            seen.add((x, y))
            com.append((x, y))
    return get_imgstack(img, np.array(com), window_size)


def imcrop_randcoord(img: np.ndarray, coord: np.ndarray, window_size: int, num_images: int,
                     random_state: int = 0):
    """`num_images` windows at distinct randomly chosen coordinates (atomai/utils/img.py:214-234)."""
    seen, com = set(), []
    while len(com) < num_images:
        i = np.random.randint(len(coord))
        if i not in seen:
            seen.add(i)
            com.append(coord[i].tolist())
    return get_imgstack(img, np.array(com), window_size)


def extract_random_subimages(imgdata: np.ndarray, window_size: int, num_images: int,
                             coordinates=None, **kwargs: int):
    """`num_images` random windows per frame, at atoms of `coord_class` or at random pixels
    (atomai/utils/img.py:237-295)."""
    from .coords import remove_edge_coord
    coord_class = kwargs.get("coord_class", 0)
    if np.ndim(imgdata) < 4:
        imgdata = imgdata[..., None]
    n = imgdata.shape[0]
    subimages_all = np.zeros((num_images * n, window_size, window_size, imgdata.shape[-1]))
    com_all = np.zeros((num_images * n, 2))
    frames_all = np.zeros((num_images * n))
    for i, img in enumerate(imgdata):
        if not coordinates:
            stack_i, com_i = imcrop_randpx(img, window_size, num_images, random_state=i)
        else:
            coord = coordinates[i]
            coord = coord[coord[:, -1] == coord_class][:, :2]
            coord = remove_edge_coord(coord, imgdata.shape[1:3], window_size // 2 + 1)
            if num_images > len(coord):
                raise ValueError("Number of images cannot be greater than the available coordinates")
            stack_i, com_i = imcrop_randcoord(img, coord, window_size, num_images, random_state=i)
        sl = slice(i * num_images, (i + 1) * num_images)
        subimages_all[sl] = stack_i
        com_all[sl] = com_i
        frames_all[sl] = np.ones(len(com_i), int) * i
    return subimages_all, com_all, frames_all


def crop_borders(imgdata: np.ndarray, thresh: float = 0) -> np.ndarray:
    """Drops the rows/columns of (h, w, c) whose values are all <= thresh, channel by channel
    (atomai/utils/img.py:502-519)."""
    out = []
    for i in range(imgdata.shape[-1]):
        img = imgdata[..., i]
        mask = img > thresh
        out.append(img[np.ix_(mask.any(1), mask.any(0))])
    return np.array(out).transpose(1, 2, 0)


def get_coord_grid(imgdata: np.ndarray, step: int, return_dict: bool = True):
    """Square grid of (row, col) points with spacing `step` for every image of a stack, in the
    Locator dictionary format or as one array (atomai/utils/img.py:522-551)."""
    if np.ndim(imgdata) == 2:
        imgdata = np.expand_dims(imgdata, axis=0)
    ii, jj = np.meshgrid(np.arange(0, imgdata.shape[1], step), np.arange(0, imgdata.shape[2], step),
                         indexing="ij")
    coord = np.stack([ii.ravel(), jj.ravel()], axis=1)
    if return_dict:
        coord = np.concatenate((coord, np.zeros((coord.shape[0], 1))), axis=-1)
        return {i: coord for i in range(imgdata.shape[0])}
    return np.concatenate([coord for _ in range(imgdata.shape[0])], axis=0)


# ------------------------------------------------------------------ bit copies on the device
# The patch gather and the lattice-mask fill copy elements bit for bit, so any numeric dtype of
# 1, 2, 4 or 8 bytes runs through one unsigned-integer kernel of that size.  A numpy array is
# uploaded once and its result copied back; a CUDA tensor stays on its device.
_BITS_NP = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}


def _is_cuda(a) -> bool:
    return hasattr(a, "is_cuda") and a.is_cuda


def _elem_bytes(dtype) -> int:
    """element size of a numpy or torch dtype the bit-copy kernels take; TypeError otherwise"""
    import torch
    if isinstance(dtype, torch.dtype):
        size = torch.empty((), dtype=dtype).element_size()
        ok = not dtype.is_complex or size <= 8
    else:
        dtype = np.dtype(dtype)
        size, ok = dtype.itemsize, dtype.kind in "biufc"
    if not ok or size not in _BITS_NP:
        raise TypeError(f"dtype {dtype} is not supported: elements must be numeric and of 1, 2, 4 "
                        "or 8 bytes")
    return size


def _device_bits(a):
    """a (numpy or CUDA) as a contiguous CUDA tensor of same-sized integers"""
    import torch
    size = _elem_bytes(a.dtype)
    if _is_cuda(a):
        return a.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32,
                                    8: torch.int64}[size])
    if not torch.cuda.is_available():
        raise RuntimeError("this function runs on a CUDA device; none is available")
    host = torch.from_numpy(np.ascontiguousarray(a).view(_BITS_NP[size]).reshape(np.shape(a)))
    return host.to("cuda")


def _from_bits(t, like):
    """a device result `t` in the dtype of `like`: a CUDA tensor, or numpy for a numpy `like`"""
    if _is_cuda(like):
        return t.view(like.dtype)
    return t.cpu().numpy().view(like.dtype)


# ------------------------------------------------------------------ random patches
# sklearn.feature_extraction.image.extract_patches_2d, which the reference calls: the same
# argument checks and errors, patch counts and draws from check_random_state, so the offsets are
# numpy's; the crops are one gather (atomai_b200_gather_patches) per image stack.
def _random_state(random_state):
    if random_state is None or random_state is np.random:
        return np.random.mtrand._rand
    if isinstance(random_state, Integral):
        return np.random.RandomState(random_state)
    if isinstance(random_state, np.random.RandomState):
        return random_state
    raise ValueError(f"{random_state!r} cannot be used to seed a numpy.random.RandomState instance")


def _check_max_patches(max_patches) -> None:
    if max_patches is None:
        return
    if isinstance(max_patches, Integral) and not isinstance(max_patches, bool):
        if max_patches >= 1:
            return
    elif isinstance(max_patches, Real) and not isinstance(max_patches, bool) and 0 < max_patches < 1:
        return
    raise ValueError("The 'max_patches' parameter must be a float in the range (0, 1), an int in "
                     f"the range [1, inf) or None. Got {max_patches!r} instead.")


def _check_image(image):
    """sklearn's check_array(allow_nd=True) for the patch source: finite, real, non-empty"""
    import torch
    if _is_cuda(image):
        if image.dtype.is_complex:
            raise ValueError("Complex data not supported")
        if image.dtype.is_floating_point and not bool(torch.isfinite(image).all()):
            raise ValueError("Input contains NaN or infinity.")
        return
    if np.iscomplexobj(image):
        raise ValueError("Complex data not supported")
    if image.dtype.kind == "f" and not np.isfinite(image).all():
        raise ValueError("Input contains NaN or infinity.")


def _patch_origins(image, patch_size, max_patches, random_state):
    """(rows, cols) of the patches extract_patches_2d takes from `image`, in its order; the
    random draws advance `random_state`'s generator as sklearn's do"""
    _check_max_patches(max_patches)
    rng = _random_state(random_state)
    i_h, i_w = image.shape[:2]
    p_h, p_w = patch_size
    if p_h > i_h:
        raise ValueError("Height of the patch should be less than the height of the image.")
    if p_w > i_w:
        raise ValueError("Width of the patch should be less than the width of the image.")
    _check_image(image)
    n_h, n_w = i_h - p_h + 1, i_w - p_w + 1
    if not max_patches:
        ii, jj = np.meshgrid(np.arange(n_h), np.arange(n_w), indexing="ij")
        return ii.ravel(), jj.ravel()
    if isinstance(max_patches, Integral):
        n = min(max_patches, n_h * n_w)
    else:
        n = int(max_patches * (n_h * n_w))    # sklearn's rounding: the product first
    i_s = rng.randint(n_h, size=n)
    j_s = rng.randint(n_w, size=n)
    return i_s, j_s


def _gather_patches(stack, origins, patch_size):
    """the patches of every frame of `stack` (f, h, w, ...) at origins [(frame, rows, cols)] as one
    gather; (K, ph, pw[, c]) in the stack's dtype, numpy or CUDA like the stack"""
    import torch
    from .. import ops
    from .graphx import _check_free
    ph, pw = patch_size
    f, h, w = stack.shape[:3]
    c = int(np.prod(stack.shape[3:], dtype=np.int64))
    size = _elem_bytes(stack.dtype)
    K = sum(len(r) for _, r, _ in origins)
    offs = np.concatenate([(k * h + rows.astype(np.int64)) * w * c + cols.astype(np.int64) * c
                           for k, rows, cols in origins]) if K else np.zeros(0, np.int64)
    out_bytes = K * ph * pw * c * size
    _check_free(out_bytes + (0 if _is_cuda(stack) else f * h * w * c * size) + 8 * K,
                "the patch gather")
    img = _device_bits(stack).reshape(f, h, w, c)
    out = torch.empty((K, ph, pw, c), dtype=img.dtype, device=img.device)
    if K:
        ops.gather_patches(img, torch.from_numpy(offs).to(img.device), ph, pw, out)
    out = _from_bits(out, stack)
    return out.reshape(K, ph, pw) if c == 1 else out


def _extract_pairs(images, masks, patch_size: int, num_patches: int, kwargs):
    """origins of every frame, images first then masks, then one gather per stack"""
    rs = kwargs.get("random_state", 0)
    if isinstance(patch_size, int):
        patch_size = (patch_size, patch_size)
    if not isinstance(patch_size, (tuple, list)):
        raise ValueError("The 'patch_size' parameter must be an instance of 'tuple' or 'list'. "
                         f"Got {patch_size!r} instead.")
    im_org, ma_org = [], []
    for k in range(min(len(images), len(masks))):
        im_org.append((k, *_patch_origins(images[k], patch_size, num_patches, rs)))
        ma_org.append((k, *_patch_origins(masks[k], patch_size, num_patches, rs)))
    if not im_org:
        raise ValueError("need at least one array to concatenate")
    return (_gather_patches(images, im_org, patch_size),
            _gather_patches(masks, ma_org, patch_size))


def extract_patches_(lattice_im, lattice_mask, patch_size: int, num_patches: int, **kwargs: int
                     ) -> Tuple[np.ndarray]:
    """Patches of `patch_size` (int: square, or (ph, pw)) from an image and its mask, as
    sklearn's extract_patches_2d takes them with max_patches=num_patches and
    random_state=kwargs.get('random_state', 0), images drawn first, then masks, from that same
    argument (atomai/utils/img.py:353-366).  Numpy arrays or CUDA tensors of any numeric dtype of
    1, 2, 4 or 8 bytes; the crops are one gather on the GPU."""
    if _is_cuda(lattice_im) is not _is_cuda(lattice_mask):
        raise TypeError("the image and the mask must both be numpy arrays or both CUDA tensors")
    if not _is_cuda(lattice_im) and not (isinstance(lattice_im, np.ndarray)
                                         and isinstance(lattice_mask, np.ndarray)):
        raise ValueError("The 'image' parameter of extract_patches_2d must be an instance of "
                         "'numpy.ndarray'")
    return _extract_pairs(lattice_im[None], lattice_mask[None], patch_size, num_patches, kwargs)


def extract_patches(images, masks, patch_size: int, num_patches: int, **kwargs: int
                    ) -> Tuple[np.ndarray]:
    """extract_patches_ on every image / mask pair of two stacks with the same arguments, in order,
    concatenated (atomai/utils/img.py:369-389); a 2-D image or mask is one frame."""
    if _is_cuda(images) is not _is_cuda(masks):
        raise TypeError("the images and the masks must both be numpy arrays or both CUDA tensors")
    if not _is_cuda(images):              # a list of frames, as np.ndim and zip take it
        images, masks = np.asarray(images), np.asarray(masks)
    if images.ndim == 2:
        images = images[None]
    if masks.ndim == 2:
        masks = masks[None]
    return _extract_pairs(images, masks, patch_size, num_patches, kwargs)


def extract_patches_and_spectra(hdata: np.ndarray, *args: np.ndarray,
                                coordinates: np.ndarray = None,
                                window_size: int = None,
                                avg_pool: int = 2,
                                **kwargs: Union[int, List[int]]
                                ) -> Tuple[np.ndarray]:
    """Image patches around `coordinates` and the spectra at their centres, from 3-D (h, w, s) or
    4-D (h, w, s1, s2) hyperspectral data (atomai/utils/img.py:392-452).  The image is args[0] or
    hdata averaged over kwargs['band'] (an int, or a 2- / 4-element list); patches come from
    extract_subimages, spectra are hdata[int(x), int(y)] of the kept coordinates, average-pooled
    over the spectral axes with kernel = stride = avg_pool by torch on the CPU.  Returns
    (patches, spectra, coordinates), the first two squeezed.  On the host: the spectra are one
    fancy-indexing gather."""
    import torch
    if hdata.ndim not in (3, 4):
        raise ValueError("Hyperspectral data must 3D or 4D")
    nspec = hdata.ndim - 2
    if args:
        img = args[0]
        if img.ndim != 2:
            raise ValueError("Image data must be 2D")
    else:
        band = kwargs.get("band", 0)
        if isinstance(band, int):
            band = [band, band + 1] * nspec
        elif nspec == 2 and isinstance(band, list) and len(band) == 2:
            band = band * 2
        window = tuple(slice(band[2 * k], band[2 * k + 1]) for k in range(nspec))
        img = hdata[(Ellipsis,) + window].mean(tuple(range(-nspec, 0)))
    patches, coords, _ = extract_subimages(img, coordinates, window_size)
    patches = patches.squeeze()
    # int() truncates toward zero, and a negative index counts from the end
    spectra = hdata[coords[:, 0].astype(np.int64), coords[:, 1].astype(np.int64)]
    pool = torch.nn.functional.avg_pool1d if nspec == 1 else torch.nn.functional.avg_pool2d
    spectra = torch.from_numpy(np.ascontiguousarray(spectra)).unsqueeze(1)
    spectra = pool(spectra, avg_pool, avg_pool).squeeze().numpy()
    return patches, spectra, coords
