"""
Coordinate utilities on the hot path's rim: centre-of-mass atom finder (Locator), the rVAE
pixel grid / rotation+translation (kept for API parity; the training path fuses the latter into
a CUDA kernel, see atomai_b200/csrc/vae.cu), atomai/utils/coords.py:21-83, and the 2-D Gaussian
peak refinement of atomai/utils/coords.py:86-231, whose fits run as one CUDA launch
(atomai_b200/csrc/refine.cu) while the O(N) bookkeeping around them stays here, and the neighbour
searches of atomai/utils/coords.py:116-515 (nearest neighbours, bond maps, predicted-to-true
pairing, clusters and trajectories through movies, DBSCAN), which run in csrc/coords.cu.
"""
import warnings
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

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


# ------------------------------------------------------------------ neighbour searches on the GPU
#
# get_nn_distances, map_bonds, compare_coordinates, find_coord_clusters, cluster_coord and
# subimg_trajectories (atomai/utils/coords.py:116-515) keep the reference's signatures and return
# values.  Their searches run in csrc/coords.cu over the cell list of csrc/graph.cu: all frames of a
# dict in one batch, float64 distances rounded as scipy's k-d tree rounds them.  One rule differs
# from the k-d tree: of two atoms at the same distance the lower index comes first (cKDTree breaks
# such ties in its own tree order).

MAX_K = 32   # _C.COORDS_MAX_K: neighbours a k-nearest search keeps in registers


def _nn_device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("the neighbour searches of utils.coords run on a CUDA device; none is "
                           "available")
    return torch.device("cuda")


def _frame_rows(coord_dict, n: int) -> np.ndarray:
    """np.append of coord_dict[0 ... n - 1] onto an empty (0, 3) float64 array, as the reference
    stacks a movie (in one concatenation)"""
    return np.concatenate([np.empty((0, 3))] + [np.asarray(coord_dict[k]) for k in range(n)], axis=0)


def _check_points(a: np.ndarray, what: str, cols=(2, 3)) -> np.ndarray:
    a = np.asarray(a)
    if a.ndim != 2 or (cols is not None and a.shape[1] not in cols) or a.shape[1] < 2:
        raise ValueError(f"{what} must be an (N, {' or '.join(map(str, cols)) if cols else '>= 2'}) "
                         f"array, got shape {a.shape}")
    if not np.isfinite(a[:, :(3 if cols else 2)]).all():
        raise ValueError(f"{what} must be finite")
    return a


def _xyz(points: np.ndarray, ncols: int = 2) -> np.ndarray:
    pos = np.zeros((len(points), 3))
    pos[:, :ncols] = points[:, :ncols]
    return pos


def _knn_side(pos: np.ndarray, nframes: int, k: int, ub: float) -> float:
    """Cell side for k-nearest searches: about max(k, 2) / 2 atoms per cell of a frame, no wider
    than an upper bound (nor narrower than 1/16 of the density side)"""
    ext = pos.max(0) - pos.min(0)
    npf = max(len(pos) / nframes, 1.0)
    span = max(float(ext[:2].max()), 1e-12)
    area = max(float(ext[0]), span / npf) * max(float(ext[1]), span / npf)
    side = float(np.sqrt(area * max(k, 2) / (2 * npf)))
    if np.isfinite(ub) and ub > 0:
        side = max(min(side, float(ub)), side / 16)
    return side


def _grid(pos: np.ndarray, side: float, nframes: int):
    """(lo, side, dims) of a cell grid over pos, with side grown until every key fits in int64"""
    lo = pos.min(0)
    while True:
        dims = np.floor((pos.max(0) - lo) / side).astype(np.int64) + 1
        if np.prod(dims.astype(np.float64)) * nframes < 2.0 ** 62 and (dims < 2 ** 31).all():
            return lo, side, dims
        side *= 2


class _Cells:
    """Points of one or more frames (stored frame by frame) in a cell grid on the device: sorted
    keys, the point of each, frame offsets and every point's cell."""

    def __init__(self, pos: np.ndarray, counts: Sequence[int], side: float, lo=None, dims=None):
        from .. import ops
        from .graphx import _check_free
        dev = _nn_device()
        N = len(pos)
        _check_free(N * 120, "the cell list")
        if lo is None:
            lo, side, dims = _grid(pos, side, len(counts))
        self.lo, self.side, self.dims = lo, side, dims
        self.pos = torch.from_numpy(np.ascontiguousarray(pos, np.float64)).to(dev)
        frame = np.repeat(np.arange(len(counts), dtype=np.int32), counts)
        self.frame = torch.from_numpy(frame).to(dev)
        self.foff = torch.from_numpy(np.concatenate(([0], np.cumsum(counts))).astype(np.int64)).to(dev)
        keys = torch.empty(N, dtype=torch.int64, device=dev)
        ops.graph_cell_keys(self.pos, self.frame, lo, side, dims, keys)
        self.keys, self.perm = torch.sort(keys, stable=True)
        self.cells = self.cells_of(self.pos)

    def cells_of(self, pos: torch.Tensor) -> torch.Tensor:
        from .. import ops
        cells = torch.empty(len(pos), 3, dtype=torch.int64, device=pos.device)
        if len(pos):
            ops.coords_cells(pos, self.lo, self.side, self.dims, cells)
        return cells

    def knn(self, qpos: torch.Tensor, qcell: torch.Tensor, qframe, k: int, ub: float):
        """(idx (Q, k) int32, dist (Q, k) float64) on the host; idx -1 / dist inf where missing"""
        from .. import ops
        from .graphx import _check_free
        Q = len(qpos)
        _check_free(Q * k * 12, "the k-nearest search")
        oidx = torch.empty(Q, k, dtype=torch.int32, device=qpos.device)
        odist = torch.empty(Q, k, dtype=torch.float64, device=qpos.device)
        ops.coords_knn(qpos, qcell, qframe, self.pos, self.keys, self.perm,
                       None if qframe is None else self.foff, self.lo, self.side, self.dims, k, ub,
                       oidx, odist)
        return oidx.cpu().numpy(), odist.cpu().numpy()


def _check_nn(nn) -> int:
    if isinstance(nn, bool) or not isinstance(nn, (int, np.integer)) or not 1 <= nn <= MAX_K - 1:
        raise ValueError(f"nn must be an integer in 1 ... {MAX_K - 1} (the k-nearest search keeps "
                         f"at most {MAX_K} atoms, the atom itself included, in registers), got {nn!r}")
    return int(nn)


def get_nn_distances(coordinates: Union[Dict[int, np.ndarray], np.ndarray], nn: int = 2,
                     upper_bound: Optional[float] = None) -> Tuple[List[np.ndarray]]:
    """
    Nearest-neighbour distances of every frame of a stack (atomai/utils/coords.py:116-149), all
    frames searched in one batch on the GPU.

    Args:
        coordinates: dict of frame -> (N, 3) arrays (x, y, class), or one such array
        nn: number of nearest neighbours, 1 ... 31
        upper_bound: only neighbours closer than this (strictly) count

    Returns:
        list of (atoms, nn) distance arrays and list of (atoms, nn + 1, 3) arrays of each atom
        with its neighbours; atoms with fewer than nn neighbours (within upper_bound) are dropped.
        An equal distance goes to the lower index.
    """
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: coordinates}
    nn = _check_nn(nn)
    ub = np.inf if upper_bound is None else float(upper_bound)
    frames = [_check_points(c, "coordinates", None) for c in coordinates.values()]
    counts = [len(c) for c in frames]
    k = nn + 1
    N = sum(counts)
    if N:
        pos = _xyz(np.concatenate([c[:, :2] for c in frames]).astype(np.float64))
        cl = _Cells(pos, counts, _knn_side(pos, len(frames), k, ub))
        idx, dist = cl.knn(cl.pos, cl.cells, cl.frame, k, ub)
    distances_all, atom_pairs_all, off = [], [], 0
    for c, n in zip(frames, counts):
        if n:
            i, d = idx[off:off + n] - off, dist[off:off + n]
            keep = (i >= 0).all(1)
            i, d = i[keep], d[keep]
        else:
            i, d = np.zeros((0, k), np.int64), np.zeros((0, k))
        distances_all.append(d[:, 1:])
        atom_pairs_all.append(c[i])
        off += n
    return distances_all, atom_pairs_all


def _pyplot():
    try:
        import matplotlib.pyplot as plt
    except ImportError:
        warnings.warn("matplotlib is not installed: plot skipped")
        return None
    return plt


def _plot_bonds(plt, distances, atom_pairs, distance_ideal, frame, show, **kwargs) -> None:
    """Bonds of every atom to its neighbours, coloured by their relative deviation from
    distance_ideal, on an h x w canvas; saved as savedir/frame_<frame>.png"""
    import os
    savedir = kwargs.get("savedir", "./")
    h, w = kwargs.get("h"), kwargs.get("w")
    if h is None or w is None:
        w = int(np.ptp(atom_pairs[..., 0])) + 10 if atom_pairs.size else 10
        h = int(np.ptp(atom_pairs[..., 1])) + 10 if atom_pairs.size else 10
    rel = (distances - distance_ideal) / distance_ideal
    fig, ax = plt.subplots(1, 1, figsize=(8, 8))
    ax.imshow(np.zeros((h, w)), cmap="gray")
    lo, hi = (float(rel.min()), float(rel.max())) if rel.size else (0.0, 1.0)
    cmap = plt.get_cmap("RdYlGn_r")
    for a, d in zip(atom_pairs, rel):
        for i in range(len(d)):
            ax.plot([a[0][1], a[i + 1][1]], [a[0][0], a[i + 1][0]],
                    c=cmap((d[i] - lo) / (hi - lo) if hi > lo else 0.5))
    ax.axis(False)
    sm = plt.cm.ScalarMappable(cmap=cmap, norm=plt.Normalize(lo, hi))
    fig.colorbar(sm, ax=ax, orientation="horizontal").set_label("Variation in bond length (%)")
    if show:
        plt.show()
    fig.savefig(os.path.join(savedir, f"frame_{frame}"))
    plt.close(fig)


def map_bonds(coordinates: Dict[int, np.ndarray], nn: int = 2, upper_bound: float = None,
              distance_ideal: float = None, plot_results: bool = True,
              **kwargs: Union[str, int]) -> np.ndarray:
    """
    Bond-length maps of a stack (atomai/utils/coords.py:475-515): the distances of every atom to
    its nn nearest neighbours, all frames searched in one batch on the GPU.  When matplotlib is
    installed, each frame's bonds are drawn coloured by their deviation from distance_ideal (by
    default the mean distance) and saved to savedir/frame_<i>.png, and shown with plot_results;
    without matplotlib the plots are skipped.  Plotting never changes the result.

    Returns:
        the concatenated (atoms, nn) distances of all frames
    """
    distances_all, atom_pairs_all = get_nn_distances(coordinates, nn, upper_bound)
    if distance_ideal is None:
        distance_ideal = np.mean(np.concatenate(distances_all))
    plt = _pyplot()
    if plt is not None:
        for i, (dist, at) in enumerate(zip(distances_all, atom_pairs_all)):
            _plot_bonds(plt, dist, at, distance_ideal, i, plot_results, **kwargs)
    return np.concatenate(distances_all)


def compare_coordinates(coordinates1: np.ndarray, coordinates2: np.ndarray, d_max: float,
                        plot_results: bool = False,
                        **kwargs: Union[int, np.ndarray]) -> Tuple[np.ndarray]:
    """
    Pairs every predicted position (coordinates1) with the nearest true one (coordinates2) and
    keeps the pairs closer than d_max (atomai/utils/coords.py:266-301).  The distance runs over all
    columns of the rows, the class column included, as the reference's k-d tree over the full rows
    does; an equal distance goes to the lower index of coordinates2.  For the plot pass the image
    as `expdata` (and `fsize`); without matplotlib it is skipped.

    Returns:
        kept rows of coordinates1, their partners in coordinates2 (both (M, 3) float64) and the
        distances (M,)
    """
    if plot_results and kwargs.get("expdata") is None:
        raise AssertionError("For plotting, provide 2D image via 'expdata' keyword")
    c1 = _check_points(coordinates1, "coordinates1")
    c2 = _check_points(coordinates2, "coordinates2")
    if c1.shape[1] != c2.shape[1]:
        raise ValueError(f"coordinates1 has {c1.shape[1]} columns, coordinates2 {c2.shape[1]}")
    ncols = c1.shape[1]
    keep, dist, idx = np.zeros(len(c1), bool), np.zeros(len(c1)), np.zeros(len(c1), np.int64)
    if len(c1) and len(c2):
        pos = _xyz(c2.astype(np.float64), ncols)
        cl = _Cells(pos, [len(pos)], _knn_side(pos, 1, 1, np.inf))
        q = torch.from_numpy(_xyz(c1.astype(np.float64), ncols)).to(cl.pos.device)
        i, d = cl.knn(q, cl.cells_of(q), None, 1, np.inf)
        idx, dist = i[:, 0], d[:, 0]
        keep = dist < d_max
    if keep.any():
        coordinates1_ = np.append(np.empty((0, 3)), c1[keep], axis=0)
        coordinates2_ = np.append(np.empty((0, 3)), c2[idx[keep]], axis=0)
    else:
        coordinates1_, coordinates2_ = np.empty((0, 3)), np.empty((0, 3))
    delta_r = dist[keep]
    if plot_results:
        plt = _pyplot()
        if plt is not None:
            fsize = kwargs.get("fsize", 20)
            plt.figure(figsize=(int(fsize * 1.25), fsize))
            plt.imshow(kwargs["expdata"], cmap="gray")
            im = plt.scatter(coordinates1_[:, 1], coordinates1_[:, 0], c=delta_r, cmap="jet", s=5)
            plt.colorbar(im).set_label("Position deviation (px)")
            plt.show()
    return coordinates1_, coordinates2_, delta_r


def _ball_side(rmax: float, span: float) -> float:
    """cell side >= rmax: two points one rmax apart land in neighbouring cells despite the few-ulp
    rounding of a cell index (as in utils.graphx), and the grid stays below 2^20 cells a side"""
    return max(rmax * (1 + 2.0 ** -48 * (span / rmax + 1)), span / 2 ** 20)


def find_coord_clusters(coord_class_dict_1: Dict[int, np.ndarray],
                        coord_class_dict_2: Dict[int, np.ndarray],
                        rmax: int) -> Tuple[np.ndarray, List]:
    """
    For every xy of coord_class_dict_1[0], the rows of coord_class_dict_2[0 ... n-1] (stacked)
    closer than rmax, in ascending distance (an equal distance goes to the lower row), with their
    xy mean and standard deviation (atomai/utils/coords.py:350-400).  One ball query on the GPU.

    Returns:
        (means (Q, 2), stds (Q, 2), list of the Q row sets)
    """
    from .. import ops
    from .graphx import _check_free, _offsets
    allc = _frame_rows(coord_class_dict_2, len(coord_class_dict_2))
    q = _check_points(np.asarray(coord_class_dict_1[0])[:, :2], "coord_class_dict_1[0]")
    _check_points(allc[:, :2], "coord_class_dict_2")
    rmax = float(rmax)
    rows = [np.zeros(0, np.int64)] * len(q)
    if len(q) and len(allc) and rmax > 0:
        pos = _xyz(allc)
        span = float((pos.max(0) - pos.min(0)).max())
        cl = _Cells(pos, [len(pos)], _ball_side(rmax, span))
        qpos = torch.from_numpy(_xyz(q.astype(np.float64))).to(cl.pos.device)
        qcell = cl.cells_of(qpos)
        args = (qpos, qcell, cl.pos, cl.keys, cl.perm, cl.lo, cl.side, cl.dims, rmax)
        cnt = torch.empty(len(q), dtype=torch.int64, device=qpos.device)
        ops.coords_ball(*args, cnt=cnt)
        rowptr = _offsets(cnt)
        M = int(rowptr[-1])
        _check_free(M * 40, "the ball query")
        oidx = torch.empty(max(M, 1), dtype=torch.int32, device=qpos.device)
        odist = torch.empty(max(M, 1), dtype=torch.float64, device=qpos.device)
        ops.coords_ball(*args, rowptr, oidx, odist)
        # each row by distance, then index: stable sorts by index, distance and row
        row = torch.repeat_interleave(torch.arange(len(q), device=qpos.device), cnt)
        o = torch.argsort(oidx[:M], stable=True)
        o = o[torch.argsort(odist[:M][o], stable=True)]
        o = o[torch.argsort(row[o], stable=True)]
        idx = oidx[:M][o].cpu().numpy()
        rp = rowptr.cpu().numpy()
        rows = [idx[rp[i]:rp[i + 1]] for i in range(len(q))]
    clusters, clusters_mean, clusters_std = [], [], []
    for r in rows:
        cluster = allc[r]
        clusters_mean.append(np.mean(cluster[:, :2], axis=0))
        clusters_std.append(np.std(cluster[:, :2], axis=0))
        clusters.append(cluster)
    return np.array(clusters_mean), np.array(clusters_std), clusters


def dbscan_labels(xy: np.ndarray, eps: float, min_samples: int) -> np.ndarray:
    """DBSCAN labels of the (N, 2) points, as sklearn's dbscan_inner assigns them: a core point has
    at least min_samples points (itself included) within eps (inclusive); clusters are the
    connected components of core points, numbered in order of their lowest core index; a border
    point joins the lowest-numbered cluster among its core neighbours; the rest is noise (-1).
    The eps-neighbourhoods come from the bond search of utils.graphx, the labels from csrc/coords.cu."""
    from .. import ops
    from .graphx import _check_free, _offsets
    dev = _nn_device()
    N = len(xy)
    pos = _xyz(np.asarray(xy, np.float64))
    span = float((pos.max(0) - pos.min(0)).max())
    side = eps * (1 + 2.0 ** -48 * (span / eps + 1))
    lo = pos.min(0)
    dims = np.floor((pos.max(0) - lo) / side).astype(np.int64) + 1
    if np.prod(dims.astype(np.float64)) >= 2.0 ** 62:
        raise ValueError("the coordinates span too many eps for the cell grid")
    _check_free(N * 64, "the DBSCAN neighbourhoods")
    t_pos = torch.from_numpy(pos).to(dev)
    keys = torch.empty(N, dtype=torch.int64, device=dev)
    ops.graph_cell_keys(t_pos, None, lo, side, dims, keys)
    keys, perm = torch.sort(keys, stable=True)
    cut = torch.full((1, 1), float(eps), dtype=torch.float64, device=dev)
    deg = torch.empty(N, dtype=torch.int32, device=dev)
    args = (t_pos, None, None, keys, perm, cut, lo, side, dims)
    ops.graph_bonds(*args, None, deg)
    rowptr = _offsets(deg)
    nnz = int(rowptr[-1])
    _check_free(nnz * 4, "the DBSCAN neighbourhoods")
    cols = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
    ops.graph_bonds(*args, rowptr, cols)
    parent = torch.empty(N, dtype=torch.int32, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    ops.coords_dbscan_roots(rowptr, cols, min_samples, parent, flag)
    rank = torch.cumsum(parent == torch.arange(N, dtype=torch.int32, device=dev), 0) - 1
    labels = torch.empty(N, dtype=torch.int64, device=dev)
    ops.coords_dbscan_labels(rowptr, cols, parent, rank, labels)
    return labels.cpu().numpy()


def cluster_coord(coord_class_dict: Dict[int, np.ndarray], eps: float,
                  min_samples: int = 10) -> Tuple[np.ndarray]:
    """
    Collapses the coordinates of a stack onto the xy plane and clusters them with DBSCAN on the
    GPU (atomai/utils/coords.py:304-347; see dbscan_labels).  Like the reference, the first entry
    of np.unique(labels) is skipped (the noise label, or cluster 0 when there is no noise).

    Returns:
        (list of the clusters' rows, cluster means (K, 2), cluster variances (K, 2))
    """
    if isinstance(eps, bool) or not isinstance(eps, (int, float, np.integer, np.floating)) or \
            not eps > 0 or not np.isfinite(eps):
        raise ValueError(f"eps must be a positive number, got {eps!r}")
    if isinstance(min_samples, bool) or not isinstance(min_samples, (int, np.integer)) or \
            min_samples < 1:
        raise ValueError(f"min_samples must be an integer >= 1, got {min_samples!r}")
    coordinates_all = _frame_rows(coord_class_dict, len(coord_class_dict))
    if len(coordinates_all) == 0:
        raise ValueError("Found array with 0 sample(s) (shape=(0, 2)) while a minimum of 1 is "
                         "required by DBSCAN.")
    _check_points(coordinates_all[:, :2], "coordinates")
    labels = dbscan_labels(coordinates_all[:, :2], float(eps), int(min_samples))
    order = np.argsort(labels, kind="stable")
    lab, starts = np.unique(labels[order], return_index=True)
    bounds = np.append(starts, len(order))
    clusters, clusters_var, clusters_mean = [], [], []
    for u in range(1, len(lab)):
        coord = coordinates_all[order[bounds[u]:bounds[u + 1]]]
        clusters.append(coord)
        clusters_mean.append(np.mean(coord[:, :2], axis=0))
        clusters_var.append(np.var(coord[:, :2], axis=0))
    return clusters, np.array(clusters_mean), np.array(clusters_var)


class subimg_trajectories:
    """
    Trajectories of single atoms or defects through a movie with the sub-images around them
    (atomai/utils/coords.py:403-472).  Every walk runs on the GPU, one thread per start position:
    in each frame (in dict order) the nearest atom closer than rmax to the walk's position (an
    equal distance goes to the lower row); when numpy's slice img[cx - r//2 : cx + r//2,
    cy - r//2 : cy + r//2] around its rounded centre is r x r, the step is recorded and the walk
    moves to that atom, else the frame is skipped.  An odd window_size therefore records nothing,
    as in the reference.  The crops are gathered on the host in one step, exact copies in the
    input's dtype.

    Args:
        imgdata: (n, h, w) or (n, h, w, c) numpy stack; frame key k crops imgdata[k]
        coord_class_dict: dict of frame -> (N, 3) coordinates
        window_size: side r of the crops
        min_length: trajectories need more than this many steps
        rmax: largest step (strict) between frames
    """

    def __init__(self, imgdata: np.ndarray, coord_class_dict: Dict[int, np.ndarray],
                 window_size: int, min_length: int = 0, rmax: int = 10) -> None:
        self.imgdata = imgdata
        self.coord_class_dict = coord_class_dict
        self.r = window_size
        self.min_length = min_length
        self.rmax = rmax

    def _walks(self, starts: np.ndarray):
        """(S, F, 4) step table (frame, atom, row0, col0), the stacked rows and the frame keys"""
        from .. import ops
        from .graphx import _check_free
        img = np.asarray(self.imgdata)
        if img.ndim not in (3, 4):
            raise ValueError(f"imgdata must be an (n, h, w) or (n, h, w, c) stack, got {img.shape}")
        if isinstance(self.r, bool) or not isinstance(self.r, (int, np.integer)):
            raise ValueError(f"window_size must be an integer, got {self.r!r}")
        keys = list(self.coord_class_dict)
        frames = [_check_points(self.coord_class_dict[k], "coordinates", None) for k in keys]
        starts = _check_points(starts, "start coordinates", (2,))
        rmax = float(self.rmax)
        counts = [len(c) for c in frames]
        F, S = len(frames), len(starts)
        rows = np.concatenate(frames) if frames else np.empty((0, 3))
        table = np.full((S, F, 4), -1, np.int64)
        table[:, :, 0] = np.arange(F)
        if S == 0 or F == 0 or sum(counts) == 0:
            return table, rows, keys
        pos = _xyz(np.concatenate([c[:, :2] for c in frames]).astype(np.float64))
        cl = _Cells(pos, counts, _knn_side(pos, F, 1, rmax))
        _check_free(S * F * 16, "the trajectory table")
        st = torch.from_numpy(_xyz(starts.astype(np.float64))).to(cl.pos.device)
        out = torch.empty(S, F, 4, dtype=torch.int32, device=cl.pos.device)
        r = int(self.r)
        ops.coords_walk(st, cl.cells_of(st), cl.pos, cl.cells, cl.keys, cl.perm, cl.foff, cl.lo,
                        cl.side, cl.dims, rmax, img.shape[1], img.shape[2], r // 2, r, out)
        return out.cpu().numpy().astype(np.int64), rows, keys

    def _collect(self, table: np.ndarray, rows: np.ndarray, keys: list):
        """(flows, frames, crops) of the walks of `table` with more than min_length steps"""
        img = np.asarray(self.imgdata)
        index = np.arange(len(img))
        fimg = np.array([index[k] for k in keys], np.int64)
        kept = [t[t[:, 1] >= 0] for t in table]
        kept = [t for t in kept if len(t) > self.min_length]
        steps = np.concatenate(kept) if kept else np.zeros((0, 4), np.int64)
        ar = np.arange(max(int(self.r), 0))
        crops = img[fimg[steps[:, 0]][:, None, None], (steps[:, 2:3] + ar)[:, :, None],
                    (steps[:, 3:4] + ar)[:, None, :]]
        flows, frames, subimgs, k = [], [], [], 0
        for t in kept:
            n = len(t)
            if n == 0:
                flows.append(np.array([]))
                frames.append(np.array([]))
                subimgs.append(np.array([]))
                continue
            flows.append(rows[t[:, 1]])
            frames.append(np.array([keys[f] for f in t[:, 0]]))
            subimgs.append(crops[k:k + n])
            k += n
        return flows, frames, subimgs

    def get_trajectory(self, img: np.ndarray, start_coord: np.ndarray) -> Tuple[np.ndarray]:
        """The trajectory from start_coord (x, y): (rows (n, 3), frame keys (n,), crops
        (n, r, r[, c])); `img` is not used, as in the reference"""
        table, rows, keys = self._walks(np.asarray(start_coord, np.float64).reshape(1, -1))
        min_length, self.min_length = self.min_length, -1
        try:
            flows, frames, subimgs = self._collect(table, rows, keys)
        finally:
            self.min_length = min_length
        return flows[0], frames[0], subimgs[0]

    def get_all_trajectories(self) -> Tuple[List[np.ndarray]]:
        """The trajectories from every atom of the first frame with more than min_length steps:
        lists of rows, frame keys and crops"""
        first = self.coord_class_dict[list(self.coord_class_dict.keys())[0]]
        table, rows, keys = self._walks(np.asarray(first)[:, :2])
        return self._collect(table, rows, keys)
