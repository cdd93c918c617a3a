"""
Host restatement of filter_cells_ / filter_cells (atomai/utils/img.py:567-625) without cv2, for
sizes beyond the goldens: the threshold as cv2.threshold applies it (float32 pixels against
float32(im_thresh)), scipy.ndimage.label with its default 4-connected cross, and the component
sizes by np.bincount.  min_index_labels gives the smallest frame-local linear index of each
pixel's component, the labels csrc/blobs.cu leaves in its workspace.
"""
import numpy as np
from scipy import ndimage


def threshold(img: np.ndarray, im_thresh: float) -> np.ndarray:
    t = np.float32(im_thresh) if img.dtype == np.float32 else np.float64(im_thresh)
    return img > t


def filter_frame(img: np.ndarray, im_thresh: float = .5, blob_thresh: float = 150,
                 filter_: str = 'below') -> np.ndarray:
    fg = threshold(img, im_thresh)
    labels, n = ndimage.label(fg)
    areas = np.bincount(labels.ravel(), minlength=n + 1).astype(np.float64)
    areas[0] = 0
    drop = areas > blob_thresh if filter_ == 'above' else areas < blob_thresh
    return (fg & ~drop[labels]).astype(np.int32)


def filter_stack(stack: np.ndarray, im_thresh: float = .5, blob_thresh: float = 50,
                 filter_: str = 'below') -> np.ndarray:
    out = np.zeros_like(stack)
    for i, img in enumerate(stack):
        out[i] = filter_frame(img, im_thresh, blob_thresh, filter_)
    return out


def min_index_labels(img: np.ndarray, im_thresh: float) -> np.ndarray:
    """int32 (h, w): the smallest linear index of each foreground pixel's component, -1 elsewhere"""
    labels, n = ndimage.label(threshold(img, im_thresh))
    _, first = np.unique(labels.ravel(), return_index=True)   # raster order: first = smallest
    if labels.min() > 0:                                       # no background pixel
        first = np.concatenate([[-1], first])
    first[0] = -1
    return first[labels].astype(np.int32)
