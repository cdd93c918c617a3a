"""
Training images from labelled ones (atomai/utils/imgen.py): a Gaussian atom and its mask on the
host, and the lattice masks that stamp a mask template at every atom of an image.  The reference
calls the mask function and assigns one slice per atom; here the mask function runs once per class
and every atom of every frame is rasterised in two GPU passes (csrc/imgen.cu): an owner pass, in
which the last atom in input order wins each pixel of its slice, and a fill pass that writes the
owners' template elements (and, for multiclass masks, the background channel).  Coordinates,
rounding, numpy's slice and broadcasting rules and every error are settled on the host first.
"""
from typing import Callable, Dict, List, Tuple, Union

import numpy as np

from .img import _device_bits, _elem_bytes, _from_bits, _is_cuda


class MakeAtom:
    """An atom modelled as a 2-D Gaussian on an sc x sc grid (sc made odd), and its mask
    (atomai/utils/imgen.py:15-79)."""

    def __init__(self, sc: int = 5, r_mask: int = 3,
                 intensity: int = 1, theta: int = 0, offset: int = 0):
        if sc % 2 == 0:
            sc += 1
        self.xo, self.yo = sc / 2, sc / 2
        axis = np.linspace(0, sc, sc)
        self.x, self.y = np.meshgrid(axis, axis)
        self.sigma_x, self.sigma_y = sc / 4, sc / 4
        self.intensity = intensity
        self.theta = theta
        self.offset = offset
        self.r_mask = r_mask

    def atom2dgaussian(self) -> np.ndarray:
        """offset + intensity exp(-(a dx² + 2 b dx dy + c dy²)), the rotated Gaussian"""
        t, sx2, sy2 = self.theta, self.sigma_x**2, self.sigma_y**2
        a = (np.cos(t)**2) / (2 * sx2) + (np.sin(t)**2) / (2 * sy2)
        b = -(np.sin(2 * t)) / (4 * sx2) + (np.sin(2 * t)) / (4 * sy2)
        c = (np.sin(t)**2) / (2 * sx2) + (np.cos(t)**2) / (2 * sy2)
        dx, dy = self.x - self.xo, self.y - self.yo
        return self.offset + self.intensity * np.exp(
            -(a * (dx**2) + 2 * b * dx * dy + c * (dy**2)))

    def circularmask(self, image: np.ndarray, radius: int) -> np.ndarray:
        """Zeroes (in place) the pixels of `image` farther than `radius` from the centre"""
        X, Y = np.ogrid[:self.x.shape[0], :self.x.shape[1]]
        dist = np.sqrt((X - self.xo + 0.5)**2 + (Y - self.yo + 0.5)**2)
        image[~(dist <= radius)] = 0
        return image

    def gen_atom_mask(self) -> Tuple[np.ndarray]:
        """(atom, mask): the mask is the atom inside radius r_mask / 2, cropped to the bounding
        box of its positive pixels, which are set to 1"""
        atom = self.atom2dgaussian()
        mask = self.circularmask(atom.copy(), self.r_mask / 2)
        rows, cols = np.nonzero(mask > 0)
        mask = mask[rows.min():rows.max() + 1, cols.min():cols.max() + 1]
        mask[mask > 0] = 1
        return atom, mask


def create_atom_mask_pair(sc: int = 5, r_mask: int = 5, intensity: int = 1):
    """(atom, mask) of MakeAtom(sc, r_mask, intensity) (atomai/utils/imgen.py:232-238)"""
    return MakeAtom(sc, r_mask, intensity).gen_atom_mask()


# ------------------------------------------------------------------ placement on the host
_CLIP = 2**40      # any rounded coordinate beyond this slices like one at it


def _slice(start: np.ndarray, stop: np.ndarray, dim: int):
    """first index and length of numpy's slice start:stop along an axis of `dim`"""
    def bound(v):
        v = np.where(v < 0, v + dim, v)
        return np.clip(v, 0, dim)
    lo, hi = bound(start), bound(stop)
    return lo, np.maximum(hi - lo, 0)


def _cast_template(mask, dtype):
    """the template in the output dtype by numpy's assignment casting (or torch's for a torch dtype
    numpy lacks), flattened, with its shape after numpy drops leading unit axes on assignment"""
    arr = np.asarray(mask)
    shape = arr.shape
    while len(shape) > 2 and shape[0] == 1:
        shape = shape[1:]
    if isinstance(dtype, np.dtype):
        out = np.empty(arr.shape, dtype)
        out[...] = arr
    else:
        import torch
        out = torch.from_numpy(np.ascontiguousarray(arr)).to(dtype)
    return out.reshape(-1), shape


class _Frame:
    """Where every atom of one frame writes: its channel, clamped slice and template strides.  The
    mask function is called once per class, in the order the classes first appear; the first
    error the reference would raise in its per-atom loop is raised here, before any device work."""

    def __init__(self, shape, xy, z, classes, make_mask, dtype):
        self.h, self.w = shape
        self.C = len(classes)
        n = len(xy)
        r = np.around(xy)
        finite = np.isfinite(r)
        stop = np.flatnonzero(~finite.all(1))
        i_round = stop[0] if len(stop) else n
        r = np.clip(np.where(finite, r, 0), -_CLIP, _CLIP).astype(np.int64)
        ch = np.searchsorted(classes, z) if self.C else np.zeros(n, np.int64)
        # mask function calls in first-appearance order, up to the first rounding failure
        called = np.unique(ch[:i_round], return_index=True)
        self.templates, sizes, shapes = [None] * self.C, np.zeros(self.C, np.int64), [None] * self.C
        i_call, err = n, None
        for c, first in sorted(zip(*called), key=lambda t: t[1]):
            try:
                _, mask = make_mask(classes[c])
                sizes[c] = mask.shape[0]
                self.templates[c], shapes[c] = _cast_template(mask, dtype)
            except Exception as e:  # raised at this class's first atom in the reference
                i_call, err = first, e
                break
            if classes[c] != classes[c]:
                # a NaN class is not a key of the reference's class-to-channel dict: KeyError at
                # its first atom, after that atom's mask function call
                i_call, err = first, KeyError(classes[c])
                break
        # numpy's slice x - r1 : x + r2 and broadcasting of the template into it
        end = min(i_round, i_call)
        size = sizes[ch[:end]]
        r1 = (size / 2 + .5).astype(np.int64)
        r2 = np.trunc(size / 2 - .5).astype(np.int64)
        self.r0, self.nr = _slice(r[:end, 0] - r1, r[:end, 0] + r2, self.h)
        self.c0, self.nc = _slice(r[:end, 1] - r1, r[:end, 1] + r2, self.w)
        th = np.array([(-1 if len(s) > 2 else 1 if len(s) < 2 else s[0]) if s is not None else 0
                       for s in shapes], np.int64)
        tw = np.array([s[-1] if s is not None else 0 for s in shapes], np.int64)
        th, tw = th[ch[:end]], tw[ch[:end]]
        fits = ((th == self.nr) | (th == 1)) & ((tw == self.nc) | (tw == 1))
        bad = np.flatnonzero(~fits)
        if len(bad):
            i = bad[0]
            raise ValueError(f"could not broadcast input array from shape {shapes[ch[i]]} into "
                             f"shape {(self.nr[i], self.nc[i])}")
        if err is not None:
            raise err
        if i_round < n:
            for v in xy[i_round]:
                int(np.around(v))
        self.ch = ch
        self.sr = np.where(th == 1, 0, tw)
        self.sc = np.where(tw == 1, 0, 1)


def _rasterise(frames: List[_Frame], dtype, background: bool, like):
    """one owner pass and one fill pass over all frames: the output of every frame, (h, w) or
    (h, w, C + 1), as consecutive views of one buffer, numpy or CUDA like `like`"""
    import torch
    from .. import _C, ops
    from .graphx import _check_free
    size = _elem_bytes(dtype)
    cout = [f.C + background if background else 1 for f in frames]
    npix = [f.h * f.w for f in frames]
    out_off = np.cumsum([0] + [p * c for p, c in zip(npix, cout)])
    own_off = np.cumsum([0] + [p * f.C for p, f in zip(npix, frames)])
    tpl_all = [t for f in frames for t in f.templates if t is not None]
    tpl_len = [len(t) if t is not None else 0 for f in frames for t in f.templates]
    tpl_off = np.cumsum([0] + tpl_len)[:-1].astype(np.int64)
    K = sum(len(f.ch) for f in frames)
    _check_free(int(out_off[-1]) * size * (1 if _is_cuda(like) else 2) + int(own_off[-1]) * 4
                + K * 4 * _C.IMGEN_ATOM_INTS + sum(tpl_len) * size, "the lattice masks")
    atoms = np.zeros((K, _C.IMGEN_ATOM_INTS), np.int64)
    k = base = 0
    for i, f in enumerate(frames):
        m = len(f.ch)
        atoms[k:k + m] = np.stack([np.full(m, i), f.ch, f.r0, f.c0, f.nr, f.nc,
                                   tpl_off[base + f.ch], f.sr, f.sc], 1)
        k, base = k + m, base + f.C
    table = np.stack([[f.h, f.w, f.C, out_off[i], own_off[i]] for i, f in enumerate(frames)])
    if tpl_all and isinstance(tpl_all[0], np.ndarray):
        tpl = _device_bits(np.concatenate(tpl_all))
    elif tpl_all:
        tpl = _device_bits(torch.cat(tpl_all).to(like.device))
    else:
        tpl = _device_bits(torch.zeros(1, dtype=dtype, device=like.device)
                           if isinstance(dtype, torch.dtype) else np.zeros(1, dtype))
    out = torch.empty(int(out_off[-1]), dtype=tpl.dtype, device=tpl.device)
    if out.numel():
        owner = torch.zeros(max(int(own_off[-1]), 1), dtype=torch.int32, device=tpl.device)
        ops.imgen_masks(torch.from_numpy(atoms.astype(np.int32)).to(tpl.device),
                        torch.from_numpy(table.astype(np.int64)).to(tpl.device), max(npix),
                        owner, tpl, out, background)
    out = out.view(torch.float64) if background else _from_bits(out, like)
    if background and not _is_cuda(like):
        out = out.cpu().numpy()
    shapes = [(f.h, f.w, c) if background else (f.h, f.w) for f, c in zip(frames, cout)]
    return out, [out[int(out_off[i]):int(out_off[i + 1])].reshape(s) for i, s in enumerate(shapes)]


def _check_rows(atoms: np.ndarray, ncols: int) -> None:
    """the error of unpacking each row into `ncols` values"""
    if atoms.ndim != 2:
        raise TypeError(f"cannot unpack non-iterable {type(atoms.flat[0]).__name__} object")
    if atoms.shape[1] > ncols:
        raise ValueError(f"too many values to unpack (expected {ncols})")
    if atoms.shape[1] < ncols:
        raise ValueError(f"not enough values to unpack (expected {ncols}, got {atoms.shape[1]})")


def _out_dtype(lattice):
    """the dtype templates are cast to: numpy's where torch's dtype has an equivalent, so numpy and
    CUDA inputs get the same bits"""
    if not _is_cuda(lattice):
        return lattice.dtype
    import torch
    try:
        return torch.empty(0, dtype=lattice.dtype).numpy().dtype
    except TypeError:
        return lattice.dtype


def _images(a):
    return a if _is_cuda(a) else np.asarray(a)


def create_lattice_mask(lattice: np.ndarray, xy_atoms: np.ndarray,
                        *args: Callable[[int, int], Tuple[np.ndarray, np.ndarray]],
                        **kwargs: int) -> np.ndarray:
    """Ground truth for one image whose atoms are all one class (atomai/utils/imgen.py:82-131):
    zeros like `lattice` (2-D, numpy or CUDA, dtype kept) with the mask of
    args[0](scale, rmask) (default create_atom_mask_pair; scale=7, rmask=5) at every (x, y) of
    `xy_atoms`, rounded half to even.  Atom x writes rows x - int(n/2 + .5) ... x + int(n/2 - .5) - 1
    of an n-row mask (columns likewise), by numpy's slice and broadcasting rules; the last atom
    wins.  The mask function is called once."""
    make_mask = args[0] if len(args) == 1 else create_atom_mask_pair
    scale, rmask = kwargs.get("scale", 7), kwargs.get("rmask", 5)
    lattice = _images(lattice)
    if len(lattice.shape) < 2:
        raise IndexError("too many indices for array")
    if len(lattice.shape) > 2:
        raise ValueError("the lattice must be a 2-D image")
    dtype = _out_dtype(lattice)
    _elem_bytes(dtype)
    xy = np.asarray(xy_atoms)
    if len(xy):
        _check_rows(xy, 2)
    else:
        xy = np.zeros((0, 2))
    frame = _Frame(tuple(lattice.shape), xy, np.zeros(len(xy)), np.zeros(1),
                   lambda z: make_mask(scale, rmask), dtype)
    return _rasterise([frame], dtype, False, lattice)[1][0]


def _multiclass_frame(shape, xyz_atoms: np.ndarray, args, kwargs) -> _Frame:
    make_mask = args[0] if len(args) == 1 else create_atom_mask_pair
    scale, rmask = kwargs.get("scale", 7), kwargs.get("rmask", 7)
    z = xyz_atoms[:, -1]
    if 0 in np.unique(z):
        xyz_atoms[:, -1] = z + 1        # in place, as the reference shifts its caller's array
    z = xyz_atoms[:, -1]
    classes = np.unique(z)
    if len(xyz_atoms):
        _check_rows(xyz_atoms, 3)
    return _Frame(shape, xyz_atoms[:, :2], z, classes,
                  lambda c: make_mask(scale, rmask, c), np.dtype(np.float64))


def create_multiclass_lattice_mask_(lattice: np.ndarray, xyz_atoms: np.ndarray,
                                    *args: Callable[[int, int], Tuple[np.ndarray, np.ndarray]],
                                    **kwargs: int) -> np.ndarray:
    """Multiclass ground truth for one image (atomai/utils/imgen.py:178-229): float64
    (h, w, C + 1), channel k the masks of args[0](scale, rmask, z) (default
    create_atom_mask_pair; scale=7, rmask=7) of the atoms of the k-th smallest class z, the last
    channel 1 - their sum, negative values set to 0.  If a class is 0, every class of `xyz_atoms`
    is raised by 1 in place.  The mask function is called once per class."""
    lattice = _images(lattice)
    frame = _multiclass_frame(tuple(lattice.shape[:2]), xyz_atoms, args, kwargs)
    return _rasterise([frame], np.dtype(np.float64), True, lattice)[1][0]


def create_multiclass_lattice_mask(imgdata: np.ndarray,
                                   coord_class_dict: Union[Dict[int, np.ndarray], np.ndarray],
                                   *args: Callable[[int, int], Tuple[np.ndarray, np.ndarray]],
                                   **kwargs: int) -> Union[List[np.ndarray], np.ndarray]:
    """create_multiclass_lattice_mask_ for every frame of a stack (a 2-D image is one frame),
    frame i with coord_class_dict[i] (an array stands for {0: array}); one stack (n, h, w, C + 1)
    when every frame has the same shape, else a list (atomai/utils/imgen.py:134-175).  All frames
    are rasterised together."""
    imgdata = _images(imgdata)
    if imgdata.ndim == 2:
        imgdata = imgdata[None]
    if isinstance(coord_class_dict, np.ndarray):
        coord_class_dict = {0: coord_class_dict}
    frames = [_multiclass_frame(tuple(img.shape[:2]), coord_class_dict[i], args, kwargs)
              for i, img in enumerate(imgdata)]
    if not frames:
        return np.array([])
    flat, masks = _rasterise(frames, np.dtype(np.float64), True, imgdata)
    if len({tuple(m.shape) for m in masks}) == 1:
        return flat.reshape(len(masks), *masks[0].shape)
    return masks
