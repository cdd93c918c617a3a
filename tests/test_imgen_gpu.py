"""utils.imgen's lattice masks and the patch gather on the GPU: every golden case bit for bit through
numpy and CUDA inputs (values, dtype, shape, array versus list, the in-place class shift, errors);
a 1024² frame of 1.6·10⁴ atoms and a 20-frame 512² stack against the host restatement
(oracle/imgen_ref.py); the last atom wins a pile-up; repeated calls give identical bits; the
training-data notebook's sequence at 512²."""
import os

import numpy as np
import pytest
import torch

import imgen_cases as ic
from atomai_b200 import utils
from oracle import imgen_ref

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda")]

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "imgen_ref.npz"))
NAMES = ("create_lattice_mask", "create_multiclass_lattice_mask", "create_multiclass_lattice_mask_",
         "extract_patches_", "extract_patches")
FNS = {n: getattr(utils, n) for n in NAMES}


def _on_cuda(fn, nimg):
    """fn with its first `nimg` arguments (images, masks) moved to the GPU"""
    def run(*args, **kwargs):
        a = [torch.from_numpy(np.ascontiguousarray(x)).cuda() if i < nimg else x
             for i, x in enumerate(args)]
        return fn(*a, **kwargs)
    return run


CUDA_FNS = {n: _on_cuda(f, 2 if n.startswith("extract") else 1) for n, f in FNS.items()}
CASES = [n for n, c in ic.all_cases().items() if c[0] in NAMES]
# cases whose images are Python lists test the numpy path's list handling; a CUDA input is a tensor
CUDA_CASES = [n for n in CASES if not isinstance(ic.all_cases()[n][1]()[0], list)]


def host(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else a


@pytest.mark.parametrize("name", CASES)
def test_goldens_numpy_inputs(name):
    ic.assert_case(GOLD, FNS, name)


@pytest.mark.parametrize("name", CUDA_CASES)
def test_goldens_cuda_inputs(name):
    ic.assert_case(GOLD, CUDA_FNS, name, host)
    if f"{name}/error" not in GOLD.files:
        res, _ = ic.call(CUDA_FNS, name)
        for t in (res if isinstance(res, (list, tuple)) else [res]):
            assert isinstance(t, torch.Tensor) and t.is_cuda


def _lattice(n, spacing, seed, classes):
    xy = ic.square(n, spacing, seed, jitter=0.4, origin=6.0)
    return ic.with_classes(xy, classes, seed)


def test_large_frame_equals_oracle():
    xyz = _lattice(126, 8.0, 1, [0, 1])                    # 15 876 atoms, 1024² frame
    img = np.zeros((1024, 1024), np.float32)
    got = utils.create_multiclass_lattice_mask_(img, xyz.copy())
    ref = imgen_ref.multiclass_mask(img.shape, xyz, utils.create_atom_mask_pair)
    assert got.tobytes() == ref.tobytes() and got.shape == ref.shape
    got = utils.create_lattice_mask(img, xyz[:, :2])
    ref = imgen_ref.lattice_mask(img, xyz[:, :2], utils.create_atom_mask_pair)
    assert got.dtype == np.float32 and got.tobytes() == ref.tobytes()


def test_stack_equals_oracle():
    rng = np.random.default_rng(2)
    d = {i: ic.with_classes(ic.square(62, 8.0, 10 + i, jitter=0.5, origin=6.0)
                            + np.array([rng.uniform(-1, 1), rng.uniform(-1, 1)]), [1, 2, 3], i)
         for i in range(20)}
    imgs = torch.zeros((20, 512, 512), device="cuda")
    got = utils.create_multiclass_lattice_mask(imgs, {k: v.copy() for k, v in d.items()})
    assert got.is_cuda and got.shape == (20, 512, 512, 4) and got.dtype == torch.float64
    ref = np.stack([imgen_ref.multiclass_mask((512, 512), d[i], utils.create_atom_mask_pair)
                    for i in range(20)])
    assert got.cpu().numpy().tobytes() == ref.tobytes()


def test_last_atom_wins():
    img = np.zeros((32, 32))
    got = utils.create_lattice_mask(img, np.array([[10.0, 10.0], [12.0, 12.0]]))
    _, t = utils.create_atom_mask_pair(7, 5)
    assert t[0, 0] == 0 and t[2, 2] == 1
    assert got[9, 9] == 0                   # the second atom's zero corner over the first's centre
    pile = np.concatenate([np.full((64, 2), 20.0), (np.arange(64) % 2)[:, None] + 1.0], 1)
    pile[::3, :2] += 0.6                    # some atoms round one pixel off
    got = utils.create_multiclass_lattice_mask_(np.zeros((40, 40)), pile.copy(),
                                                lambda s, r, z: (None, ic.asym_mask(s, r, z)[1]))
    ref = imgen_ref.multiclass_mask((40, 40), pile, lambda s, r, z: (None, ic.asym_mask(s, r, z)[1]))
    assert got.tobytes() == ref.tobytes()


def test_repeat_calls_identical():
    xyz = _lattice(60, 4.0, 3, [0, 1, 2])
    img = torch.zeros((256, 256), device="cuda")
    a = utils.create_multiclass_lattice_mask_(img, xyz.copy())
    b = utils.create_multiclass_lattice_mask_(img, xyz.copy())
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_notebook_sequence_512():
    rng = np.random.default_rng(5)
    lattice_im = rng.random((512, 512))
    xy1 = ic.square(63, 8.0, 6, jitter=0.4, origin=6.0)
    xy2 = xy1[::3] + 4.0
    m1 = utils.create_lattice_mask(lattice_im, xy1)
    m2 = utils.create_lattice_mask(lattice_im, xy2, scale=9, rmask=7)
    r1 = imgen_ref.lattice_mask(lattice_im, xy1, utils.create_atom_mask_pair)
    r2 = imgen_ref.lattice_mask(lattice_im, xy2, utils.create_atom_mask_pair, 9, 7)
    assert m1.tobytes() == r1.tobytes() and m2.tobytes() == r2.tobytes()
    bg = 1 - (m1 + m2)
    bg[bg < 0] = 0
    mask = np.stack([m1, m2, bg], -1)
    images, labels = utils.extract_patches_(lattice_im, mask, 256, 100, random_state=42)
    rs = np.random.RandomState(42)
    i, j = rs.randint(257, size=100), rs.randint(257, size=100)
    ref_im = np.stack([lattice_im[a:a + 256, b:b + 256] for a, b in zip(i, j)])
    ref_lb = np.stack([mask[a:a + 256, b:b + 256] for a, b in zip(i, j)])
    assert images.tobytes() == ref_im.tobytes() and labels.tobytes() == ref_lb.tobytes()
    assert images.shape == (100, 256, 256) and labels.shape == (100, 256, 256, 3)


def test_subimages_gather_unchanged():
    rng = np.random.default_rng(9)
    stack = rng.random((3, 64, 64, 2)).astype(np.float32)
    stack[1, 30, 30, 1] = np.nan
    coords = {i: ic.with_classes(rng.uniform(-3, 66, (40, 2)), [0], i) for i in range(3)}
    ref = utils.extract_subimages(stack, coords, 9)
    got = utils.extract_subimages(torch.from_numpy(stack).cuda(), coords, 9)
    assert got[0].cpu().numpy().tobytes() == ref[0].tobytes()
    np.testing.assert_array_equal(got[1], ref[1])
    np.testing.assert_array_equal(got[2], ref[2])
