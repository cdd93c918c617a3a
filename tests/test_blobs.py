"""filter_cells / filter_cells_ without a GPU: the host restatement (oracle/blobs_ref.py) reproduces
the reference's outputs in tests/golden/blobs_ref.npz exactly; the public signatures are the
reference's; every documented error is raised before any device work."""
import inspect
import os

import numpy as np
import pytest
import torch

import blobs_cases as bc
from atomai_b200 import ops, utils
from atomai_b200.utils import graphx, img
from oracle import blobs_ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blobs_ref.npz"))
ORACLE = {"filter_cells_": blobs_ref.filter_frame, "filter_cells": blobs_ref.filter_stack}
OUT_CASES = [n for n in bc.all_cases() if f"{n}/out" in GOLD.files]
ERROR_CASES = [n for n in bc.all_cases() if f"{n}/error" in GOLD.files]


def test_every_case_has_a_golden():
    assert len(OUT_CASES) + len(ERROR_CASES) == len(bc.all_cases())


@pytest.mark.parametrize("name", OUT_CASES)
def test_oracle_equals_goldens(name):
    got, ref = bc.call(ORACLE, name), GOLD[f"{name}/out"]
    assert got.shape == ref.shape and got.dtype == ref.dtype
    assert np.array_equal(got, ref)


def test_min_index_labels():
    im = np.array([[1, 0, 1, 1],
                   [1, 0, 0, 1],
                   [1, 1, 0, 1],
                   [0, 0, 1, 0]], np.float32)
    want = np.array([[0, -1, 2, 2],
                     [0, -1, -1, 2],
                     [0, 0, -1, 2],
                     [-1, -1, 14, -1]], np.int32)
    assert np.array_equal(blobs_ref.min_index_labels(im, .5), want)
    assert np.array_equal(blobs_ref.min_index_labels(np.ones((2, 3)), .5), np.zeros((2, 3)))


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(ops, "blob_filter", fail)
    monkeypatch.setattr(graphx, "_check_free", fail)
    monkeypatch.setattr(torch.Tensor, "to", fail)


@pytest.mark.parametrize("name", ERROR_CASES)
def test_golden_errors_before_device_work(monkeypatch, name):
    _no_device(monkeypatch)
    with pytest.raises(bc.expected_error(str(GOLD[f"{name}/error"]))):
        bc.call(utils, name)


@pytest.mark.parametrize("call, err", [
    (lambda: utils.filter_cells_(np.ones((2, 4, 4), np.float32)), ValueError),
    (lambda: utils.filter_cells_(np.ones(4, np.float32)), ValueError),
    (lambda: utils.filter_cells(np.ones((4, 4), np.float32)), ValueError),
    (lambda: utils.filter_cells(np.ones((1, 2, 4, 4), np.float32)), ValueError),
    (lambda: utils.filter_cells_(np.ones((4, 4)), im_thresh=np.nan), ValueError),
    (lambda: utils.filter_cells_(np.ones((4, 4)), im_thresh=np.inf), ValueError),
    (lambda: utils.filter_cells(np.ones((2, 4, 4)), im_thresh=-np.inf), ValueError),
    (lambda: utils.filter_cells_(np.ones((4, 4)), im_thresh="0.5"), TypeError),
    (lambda: utils.filter_cells_(np.ones((4, 4)), blob_thresh="3"), TypeError),
    (lambda: utils.filter_cells_(np.ones((4, 4)), blob_thresh=np.ones(2)), TypeError),
    (lambda: utils.filter_cells_([[1.0, 0.0]]), TypeError),
    (lambda: utils.filter_cells_(torch.ones(4, 4)), TypeError),            # a CPU tensor
    (lambda: utils.filter_cells(np.ones((2, 4, 4), np.uint32)), TypeError),
    (lambda: utils.filter_cells(np.ones((2, 4, 4), np.complex64)), TypeError),
    (lambda: utils.filter_cells(np.zeros((0, 4, 4), np.int8)), TypeError),  # checked when empty too
    (lambda: utils.filter_cells(np.zeros((0, 4, 4)), im_thresh=np.nan), ValueError),
])
def test_documented_errors_before_device_work(monkeypatch, call, err):
    _no_device(monkeypatch)
    with pytest.raises(err):
        call()


def test_frame_of_2_31_pixels_raises(monkeypatch):
    _no_device(monkeypatch)
    big = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), (2**16, 2**15), (0, 0))
    with pytest.raises(ValueError):
        utils.filter_cells_(big)
    with pytest.raises(ValueError):
        utils.filter_cells(big[None])
    empty = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), (0, 2**16, 2**15), (0, 0, 0))
    with pytest.raises(ValueError):
        utils.filter_cells(empty)


def test_working_set_beyond_free_memory_raises(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device work after the memory check")
    monkeypatch.setattr(ops, "blob_filter", fail)
    monkeypatch.setattr(torch.Tensor, "to", fail)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 1 << 30))
    with pytest.raises(MemoryError):
        utils.filter_cells(np.zeros((4, 256, 256), np.float32))


def test_empty_stack_needs_no_device(monkeypatch):
    _no_device(monkeypatch)
    for dt in bc.ACCEPTED:
        out = utils.filter_cells(np.zeros((0, 3, 5), dt))
        assert out.shape == (0, 3, 5) and out.dtype == dt


def test_signatures_equal_the_reference():
    ref = {
        "filter_cells_": "(imgdata, im_thresh=0.5, blob_thresh=150, filter_='below')",
        "filter_cells": "(imgdata, im_thresh=0.5, blob_thresh=50, filter_='below')",
    }
    for name, sig in ref.items():
        f = getattr(utils, name)
        assert f is getattr(img, name)
        s = inspect.signature(f)
        plain = s.replace(parameters=[p.replace(annotation=p.empty) for p in s.parameters.values()],
                          return_annotation=s.empty)
        assert str(plain) == sig, name
