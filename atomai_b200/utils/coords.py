"""
Coordinate utilities on the hot path's rim: centre-of-mass atom finder (Locator), the rVAE
pixel grid / rotation+translation (kept for API parity; the training path fuses the latter into
a CUDA kernel, see atomai_b200/csrc/vae.cu), atomai/utils/coords.py:21-83, and the 2-D Gaussian
peak refinement of atomai/utils/coords.py:86-231, whose fits run as one CUDA launch
(atomai_b200/csrc/refine.cu) while the O(N) bookkeeping around them stays here.
"""
import warnings
from typing import Callable, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from scipy import ndimage, spatial


def find_com(image_data: np.ndarray) -> np.ndarray:
    """Centres of mass of the 4-connected blobs of a thresholded image
    (atomai/utils/coords.py:21-34)."""
    labels, nlabels = ndimage.label(image_data)
    coordinates = np.array(
        ndimage.center_of_mass(image_data, labels, np.arange(nlabels) + 1))
    return coordinates.reshape(coordinates.shape[0], 2)


def grid2xy(X1: torch.Tensor, X2: torch.Tensor) -> torch.Tensor:
    """(M, N) grids -> (M*N, 2) xy coordinates (atomai/utils/coords.py:37-44)."""
    X = torch.stack((X1, X2), 0)
    return X.reshape(2, -1).T


def imcoordgrid(im_dim: Tuple) -> torch.Tensor:
    """Pixel-coordinate grid in [-1, 1]: x (slow axis) ascending, y descending
    (atomai/utils/coords.py:47-54)."""
    xx = torch.linspace(-1, 1, im_dim[0])
    yy = torch.linspace(1, -1, im_dim[1])
    x0, x1 = torch.meshgrid(xx, yy, indexing="ij")
    return grid2xy(x0, x1)


def transform_coordinates(coord: Union[np.ndarray, torch.Tensor],
                          phi: torch.Tensor,
                          coord_dx: Union[np.ndarray, torch.Tensor, int] = 0) -> torch.Tensor:
    """Batched 2-D rotation followed by translation: coord @ [[c, s], [-s, c]] + dx
    (atomai/utils/coords.py:57-83).  Plain torch; used outside the fused training kernel."""
    if isinstance(coord, np.ndarray):
        coord = torch.from_numpy(coord).float()
    if isinstance(coord_dx, np.ndarray):
        coord_dx = torch.from_numpy(coord_dx).float()
    c, s = torch.cos(phi), torch.sin(phi)
    rot = torch.stack([torch.stack([c, s], 1), torch.stack([-s, c], 1)], 1)
    return torch.bmm(coord, rot) + coord_dx


def remove_edge_coord(coordinates: np.ndarray, dim: Tuple, dist_edge: int) -> np.ndarray:
    """Drops the coordinates closer than `dist_edge` to an image edge
    (atomai/utils/coords.py:518-537; note the reference compares column 0 with the WIDTH and
    column 1 with the HEIGHT — kept)."""
    h, w = dim
    c = np.asarray(coordinates)
    if len(c) == 0:
        return coordinates
    bad = (c[:, 0] > w - dist_edge) | (c[:, 0] < dist_edge) | (c[:, 1] > h - dist_edge) | (c[:, 1] < dist_edge)
    return c[~bad]


REFINE_D_MAX = 16   # windows up to 32 x 32: the m x 7 Jacobian of a fit lives in shared memory


def get_nn_distances_(coordinates: np.ndarray, nn: int = 2,
                      upper_bound: Optional[float] = None) -> Tuple[np.ndarray]:
    """Distances to the `nn` nearest neighbours of every atom of one frame and the coordinates of
    each atom with its neighbours (atomai/utils/coords.py:86-113); atoms without `nn` neighbours
    within `upper_bound` are dropped."""
    upper_bound = np.inf if upper_bound is None else upper_bound
    tree = spatial.cKDTree(coordinates[:, :2])
    dist, idx = tree.query(coordinates[:, :2], k=nn + 1, distance_upper_bound=upper_bound)
    missing = np.where(dist == np.inf)[0]
    idx = np.delete(idx, missing, axis=0)
    dist = np.delete(dist, missing, axis=0)
    return dist[:, 1:], coordinates[idx]


def _default_d(coordinates: np.ndarray) -> int:
    """1/4 of the mean distance to the two nearest neighbours (coords.py:200-207)."""
    warnings.warn(
        "The d-value for bounding box not found. Defaulting to 1/4 of mean atomic distance.",
        stacklevel=3)
    dist = np.concatenate(get_nn_distances_(coordinates)[0])
    return int(np.mean(dist) * 0.25)


def _slice_bound(i: np.ndarray, length: int) -> np.ndarray:
    """A slice bound as numpy resolves it for a positive step."""
    return np.clip(np.where(i < 0, i + length, i), 0, length)


def _window_origins(shape: Tuple[int, int], coordinates: np.ndarray, d: int) -> np.ndarray:
    """(N, 2) int top-left corners of img[cx-d:cx+d, cy-d:cy+d], cx, cy = int(np.around(c)), or -1
    where numpy's slice of that window is not (2d, 2d) and the atom keeps its position."""
    c = np.around(coordinates[:, :2]).astype(np.int64)
    out = np.full(c.shape, -1, np.int64)
    full = np.ones(len(c), bool)
    for ax in range(2):
        start = _slice_bound(c[:, ax] - d, shape[ax])
        stop = _slice_bound(c[:, ax] + d, shape[ax])
        full &= np.maximum(stop - start, 0) == 2 * d
        out[:, ax] = start
    out[~full] = -1
    return out


def _fit_native(stack: Union[np.ndarray, torch.Tensor], table: np.ndarray,
                dmax: int) -> Tuple[np.ndarray, np.ndarray]:
    """All fits of the (K, 4) int32 table {frame, row0, col0, d} in one launch over the (n, H, W)
    stack: one upload, one download.  Returns popt (K, 7) float64 and info (K,) int32."""
    from .. import ops
    if isinstance(stack, torch.Tensor) and stack.is_cuda:
        dev = stack.device
        stack = stack.detach().float().contiguous()
    else:
        if not torch.cuda.is_available():
            raise RuntimeError("peak refinement runs on CUDA (sm_90a) only; there is no CPU path")
        dev = torch.device("cuda", torch.cuda.current_device())
        stack = torch.as_tensor(np.ascontiguousarray(stack, np.float32)).to(dev)
    with torch.cuda.device(dev):
        atoms = torch.from_numpy(np.ascontiguousarray(table, np.int32)).to(dev)
        popt = torch.empty((len(table), 7), dtype=torch.float64, device=dev)
        info = torch.empty(len(table), dtype=torch.int32, device=dev)
        ops.peak_refine(stack, atoms, dmax, popt, info)
        out = torch.cat([popt, info.double()[:, None]], 1).cpu().numpy()
    return out[:, :7], out[:, 7].astype(np.int32)


def refine_frames(images: Union[np.ndarray, torch.Tensor], coordinates: Sequence[np.ndarray],
                  d: Optional[int] = None, fit: Optional[Callable] = None) -> List[np.ndarray]:
    """peak_refinement of every frame of an (n, H, W) stack with its (N_i, 3) coordinates, all fits
    in one launch.  d=None: each frame's default d.  `fit(images, table, dmax) -> (popt, info)`
    replaces the native fits (the parity tests pass the scipy oracle)."""
    from .._C import REFINE_NONFINITE
    h, w = images.shape[-2:]
    tables, ds = [], []
    for i, c in enumerate(coordinates):
        c = np.asarray(c)
        di = d
        if di is None and len(c):
            di = _default_d(c)
        di = 1 if di is None else int(di)
        if not 1 <= di <= REFINE_D_MAX:
            raise ValueError(f"peak refinement supports 1 <= d <= {REFINE_D_MAX}, got d={di}")
        org = _window_origins((h, w), c, di)
        t = np.empty((len(c), 4), np.int64)
        t[:, 0], t[:, 1:3], t[:, 3] = i, org, di
        t[org[:, 0] < 0, 1:3] = -1
        tables.append(t)
        ds.append(di)
    table = np.concatenate(tables) if tables else np.empty((0, 4), np.int64)
    fitted = table[:, 1] >= 0
    popt = np.full((len(table), 7), np.nan)
    info = np.full(len(table), -1, np.int32)
    if fitted.any():
        popt[fitted], info[fitted] = (fit or _fit_native)(images, table[fitted].astype(np.int32),
                                                          max(ds))
    if (info == REFINE_NONFINITE).any():
        raise ValueError("array must not contain infs or NaNs")
    if (info[fitted] == 0).any():
        raise TypeError("The number of func parameters=7 must not exceed the number of data "
                        f"points={4 * int(table[fitted][info[fitted] == 0, 3][0]) ** 2}")
    out, k = [], 0
    for c, di in zip(coordinates, ds):
        c = np.asarray(c)
        sl = slice(k, k + len(c))
        k += len(c)
        out.append(_finish(c, di, popt[sl], info[sl]))
    return out


def _finish(coordinates: np.ndarray, d: int, popt: np.ndarray, info: np.ndarray) -> np.ndarray:
    """Steps after the fits (coords.py:220-231): a converged fit (info 1-4) whose centre lies
    within 3 px of the window centre moves the atom to popt[1:3] + np.around(c) - d; every other
    atom keeps c.  The class column is carried over."""
    xy = np.array(coordinates[:, :2], np.float64)
    if len(xy) == 0:
        return np.empty((0, 3))
    ctr = popt[:, 1:3] - d
    r = np.sqrt(ctr[:, 0] * ctr[:, 0] + ctr[:, 1] * ctr[:, 1])
    accept = (info >= 1) & (info <= 4) & (r < 3)
    # borderline radii: decide with the reference's own expression
    for i in np.where((info >= 1) & (info <= 4) & (np.abs(r - 3) < 1e-9))[0]:
        accept[i] = np.linalg.norm(popt[i, 1:3] - d) < 3
    xy[accept] = popt[accept, 1:3] + np.around(coordinates[accept, :2]) - d
    return np.concatenate((xy, coordinates[:, 2:3]), axis=-1)


def peak_refinement(imgdata: Union[np.ndarray, torch.Tensor], coordinates: np.ndarray,
                    d: Optional[int] = None) -> np.ndarray:
    """
    Refines atomic positions by fitting a 2-D Gaussian around each one, with the neural-network
    positions as the initial guess (atomai/utils/coords.py:179-231).

    Args:
        imgdata: single (H, W) image, numpy or CUDA tensor; fitted in float64 from its float32
            values
        coordinates: (N, 3) array: x, y (row, column) and atom class
        d: half-side of the fitted square, 1 <= d <= 16; by default 1/4 of the mean
            nearest-neighbour distance

    Returns:
        (N, 3) array of refined coordinates
    """
    stack = imgdata[None] if isinstance(imgdata, torch.Tensor) else np.asarray(imgdata)[None]
    return refine_frames(stack, [np.asarray(coordinates)], d)[0]


def get_lengthscale_constraints(grid: np.ndarray) -> list:
    """[lower, upper] lengthscale bounds for a GP on the pixel grid `grid` ((N, ndim) indices):
    1 and half the largest index + 1 per dimension (atomai/utils/coords.py:540-543)."""
    upper = np.amax(grid, axis=0) // 2 + 1
    return [np.ones(grid.shape[-1]).tolist(), upper.tolist()]


def get_intensities(coordinates_all: dict, nn_input: np.ndarray, r: int = 3) -> List[np.ndarray]:
    """Mean intensity of the r x r square (rows and columns from x - r//2, odd r centred) around
    the rounded (x, y) of every atom, one array per frame key of `coordinates_all`, with frame k
    taken from nn_input[k] (atomai/utils/coords.py:234-275)."""
    out = []
    h = r // 2
    hi = h + 1 if r % 2 else h
    for k, coord in coordinates_all.items():
        img = nn_input[k]
        vals = []
        for c in coord:
            cx, cy = int(np.around(c[0])), int(np.around(c[1]))
            vals.append(np.mean(img[cx - h:cx + hi, cy - h:cy + hi]))
        out.append(np.array(vals))
    return out
