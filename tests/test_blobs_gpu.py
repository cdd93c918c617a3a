"""filter_cells / filter_cells_ on the GPU: every golden case through numpy and CUDA inputs equals
the reference exactly (values, dtype, shape, errors); a 64-frame 1024² stack and 4096² frames at
fill fractions 0.3, 0.59 (near the square lattice's site-percolation threshold, where the largest
components are fractal and span many tiles) and 0.8 equal the host restatement
(oracle/blobs_ref.py); the label workspace holds each component's smallest frame-local index;
repeated calls give identical bits."""
import os

import numpy as np
import pytest
import torch

import blobs_cases as bc
from atomai_b200 import ops, utils
from oracle import blobs_ref

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda")]

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blobs_ref.npz"))
CASES = list(bc.all_cases())


def _cuda_fns():
    def wrap(f):
        return lambda x, *a, **k: f(torch.from_numpy(np.ascontiguousarray(x)).cuda(), *a, **k)
    return {n: wrap(getattr(utils, n)) for n in ("filter_cells_", "filter_cells")}


def _check(name, fns, cuda_out):
    if f"{name}/error" in GOLD.files:
        with pytest.raises(bc.expected_error(str(GOLD[f"{name}/error"]))):
            bc.call(fns, name)
        return
    got = bc.call(fns, name)
    if cuda_out:
        assert isinstance(got, torch.Tensor) and got.is_cuda
        got = got.cpu().numpy()
    ref = GOLD[f"{name}/out"]
    assert isinstance(got, np.ndarray) and got.shape == ref.shape and got.dtype == ref.dtype
    assert np.array_equal(got, ref), name


@pytest.mark.parametrize("name", CASES)
def test_goldens_numpy_inputs(name):
    _check(name, utils, False)


@pytest.mark.parametrize("name", CASES)
def test_goldens_cuda_inputs(name):
    _check(name, _cuda_fns(), True)


def test_stack_64x1024_equals_oracle():
    st = bc.stack(64, 1024, 1024, 100, 0.45)
    got = utils.filter_cells(st, im_thresh=0.55, blob_thresh=20)
    ref = blobs_ref.filter_stack(st, 0.55, 20)
    assert got.dtype == np.float32 and np.array_equal(got, ref)
    got = utils.filter_cells(torch.from_numpy(st).cuda(), 0.55, 20, 'above')
    assert np.array_equal(got.cpu().numpy(), blobs_ref.filter_stack(st, 0.55, 20, 'above'))


@pytest.mark.parametrize("fill", [0.3, 0.59, 0.8])
def test_4096_frame_equals_oracle(fill):
    im = bc.field(4096, 4096, 200, fill)
    for bt, f in ((20, "below"), (1000, "above")):
        got = utils.filter_cells_(im, 1 - fill, bt, f)
        ref = blobs_ref.filter_frame(im, 1 - fill, bt, f)
        assert got.dtype == np.int32 and np.array_equal(got, ref), (bt, f)


def _labels(st, im_thresh, blob_thresh=0.0, above=False):
    x = torch.from_numpy(st).cuda()
    labels = torch.empty(x.shape, dtype=torch.int32, device="cuda")
    counts = torch.empty_like(labels)
    out = torch.empty(x.shape, dtype=torch.int32, device="cuda")
    ops.blob_filter(x, im_thresh, blob_thresh, above, labels, counts, out)
    return labels.cpu().numpy(), counts.cpu().numpy(), out.cpu().numpy()


@pytest.mark.parametrize("kind", ["field", "snake", "comb"])
def test_label_workspace_is_the_smallest_index(kind):
    if kind == "field":
        st = np.stack([bc.field(300, 517, 300 + i, 0.59) for i in range(3)])
    elif kind == "snake":
        st = np.stack([bc.snake(300, 517), bc.snake(517, 300, True)])
    else:
        st = np.stack([bc.comb(300, 517), bc.comb(517, 300).T.copy()])
    th = 0.41 if kind == "field" else 0.5
    labels, counts, _ = _labels(st, th)
    for k, im in enumerate(st):
        want = blobs_ref.min_index_labels(im, th)
        assert np.array_equal(labels[k], want), k
        # and the count at each root is its component's size
        roots, sizes = np.unique(want[want >= 0], return_counts=True)
        assert np.array_equal(counts[k].ravel()[roots], sizes)


def test_repeat_calls_identical():
    st = bc.stack(4, 1024, 1024, 500, 0.59)
    a = _labels(st, 0.41, 30.0)
    b = _labels(st, 0.41, 30.0)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    x = torch.from_numpy(st).cuda()
    assert torch.equal(utils.filter_cells(x, 0.41, 30), utils.filter_cells(x, 0.41, 30))
