"""FFTmask / FFTsub / threshImg without a GPU: the float64 host restatement (oracle/fft_ref.py)
reproduces the reference's outputs in tests/golden/fft_ref.npz within the bounds of
fft_cases.py; the public signatures are the reference's; every documented error is raised
before any device work."""
import inspect
import os

import numpy as np
import pytest
import torch

import fft_cases as fc
from atomai_b200 import ops, utils
from atomai_b200.utils import graphx, img
from oracle import fft_ref

GOLD = fc.load_golden(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                    "fft_ref.npz"))
ORACLE = {"FFTmask": fft_ref.fftmask, "FFTsub": fft_ref.fftsub, "threshImg": fft_ref.threshimg}
CASES = fc.all_cases()
ERROR_CASES = [n for n in CASES if f"{n}/error" in GOLD.files]
OUT_CASES = [n for n in CASES if n not in ERROR_CASES]


def gold(key):
    return GOLD[key]


def test_every_case_has_a_golden():
    for n in OUT_CASES:
        assert all(f"{n}/{k}" in GOLD.files for k in fc.result_keys(n)), n


def check_against_gold(name, got):
    """got: the results of case `name` as numpy arrays; compares them with the goldens"""
    fn, args, _ = CASES[name]
    refs = [GOLD[f"{name}/{k}"] for k in fc.result_keys(name)]
    assert len(got) == len(refs)
    for g, r in zip(got, refs):
        assert isinstance(g, np.ndarray) and g.dtype == r.dtype and g.shape == r.shape, name
    if fn == "threshImg":
        assert np.array_equal(got[0], refs[0])
        return
    if fn == "FFTmask":
        F2, F3 = got
        R2, R3 = refs
        if not np.isfinite(R2).all():
            assert not np.isfinite(F2).any() and not np.isfinite(F3).any()
            return
        single = R2.dtype == np.complex64
        for g, r in ((F2, R2), (F3, R3)):
            assert np.linalg.norm((g.astype(np.complex128) - r)) <= fc.spectrum_tol(r, single)
        assert np.array_equal(fc.masked(F2, F3), fc.masked(R2, R3))
        return
    src, spec = args(gold)
    ref = refs[0]
    if not np.isfinite(src).all():
        # a NaN pixel makes the minimum NaN; an inf pixel makes the range inf: 0 on finite
        # pixels, NaN on the inf one
        assert np.array_equal(got[0], ref, equal_nan=True)
        return
    if name.startswith("sub_const"):
        assert np.isnan(got[0]).all() and np.isnan(ref).all()
        return
    _, raw = fft_ref.fftsub(src, spec, raw=True)
    tol = fc.sub_tol(src, spec, raw, spec.dtype == np.complex64)
    if name.startswith("sub_noise"):
        assert tol is None
    if tol is None:
        # rounding noise, or an exactly constant difference (a 1 x 1 image): 0 / 0
        assert np.isnan(got[0]).all() or (np.isfinite(got[0]).all() and got[0].min() >= 0
                                          and got[0].max() <= 1)
        return
    assert np.abs(got[0].astype(np.float64) - ref).max() <= tol, name


@pytest.mark.parametrize("name", OUT_CASES)
def test_oracle_reproduces_goldens(name):
    got = fc.call(ORACLE, name, gold)
    check_against_gold(name, got if isinstance(got, tuple) else (got,))


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device work before the argument checks")
    monkeypatch.setattr(ops, "fft2_mask", fail)
    monkeypatch.setattr(ops, "fft2_sub", fail)
    monkeypatch.setattr(graphx, "_check_free", fail)
    monkeypatch.setattr(torch.Tensor, "to", fail)


@pytest.mark.parametrize("name", ERROR_CASES)
def test_golden_errors_before_device_work(monkeypatch, name):
    import builtins
    _no_device(monkeypatch)
    with pytest.raises(getattr(builtins, str(GOLD[f"{name}/error"]))):
        fc.call(utils, name, gold)


def _big(h, w, dtype=np.float32):
    return np.lib.stride_tricks.as_strided(np.zeros(1, dtype), (h, w), (0, 0))


F64 = np.ones((8, 8))
C128 = np.ones((8, 8), np.complex128)


@pytest.mark.parametrize("call, err", [
    (lambda: utils.FFTmask(_big(4097, 8)), ValueError),
    (lambda: utils.FFTmask(_big(8, 4097)), ValueError),
    (lambda: utils.FFTmask(_big(6000, 16)), ValueError),
    (lambda: utils.FFTmask(_big(16384, 16384)), ValueError),
    (lambda: utils.FFTmask(_big(8192, 12288)), ValueError),
    (lambda: utils.FFTsub(_big(4097, 64), _big(4097, 64, np.complex64)), ValueError),
    (lambda: utils.FFTmask(np.ones((2, 8, 8))), ValueError),
    (lambda: utils.FFTmask(np.ones((8, 8)), maskratio=0), ZeroDivisionError),
    (lambda: utils.FFTmask(np.ones((128, 40))), ValueError),
    (lambda: utils.FFTmask(np.ones((64, 64)), maskratio=1), ValueError),
    (lambda: utils.FFTmask(np.ones((8, 8), np.longdouble)), TypeError),
    (lambda: utils.FFTmask(np.ones((8, 8), np.clongdouble)), TypeError),
    (lambda: utils.FFTmask(np.ones((8, 8), object)), TypeError),
    (lambda: utils.FFTmask(np.array([["a", "b"]])), TypeError),
    (lambda: utils.FFTmask([[1.0, 2.0]]), TypeError),
    (lambda: utils.FFTmask(torch.ones(8, 8)), TypeError),                  # a CPU tensor
    (lambda: utils.FFTsub(F64, F64), TypeError),                            # a real spectrum
    (lambda: utils.FFTsub(F64, np.ones((8, 8), np.clongdouble)), TypeError),
    (lambda: utils.FFTsub(np.ones((8, 8), np.longdouble), C128), TypeError),
    (lambda: utils.FFTsub(F64, np.ones((8, 7), np.complex128)), ValueError),
    (lambda: utils.FFTsub(np.ones(8), np.ones(8, np.complex128)), ValueError),
    (lambda: utils.FFTsub(F64, C128[None]), ValueError),
])
def test_documented_errors_before_device_work(monkeypatch, call, err):
    _no_device(monkeypatch)
    with pytest.raises(err):
        call()


def test_size_limits():
    from atomai_b200 import _C
    for n in (1, 2, 97, 4093, 4096, 8192):
        assert img._fft_shape((n, 5)) == (n, 5)
        assert ops.fft2_workspace_bytes(n, 5) > 0
    for n in (4097, 6000, 8191, 16384):
        assert ops.fft2_workspace_bytes(n, 5) == -1
        with pytest.raises(ValueError):
            img._fft_shape((5, n))
    assert _C.FFT_MAX_SIDE == 4096 and _C.FFT_MAX_POW2 == 8192


def test_mask_box_follows_numpy_slices():
    assert img._mask_box((64, 64), 10) == (26, 26, 6)
    assert img._mask_box((33, 50), 4) == (8, 8, 8)
    assert img._mask_box((64, 64), 2) == (0, 0, 32)
    assert img._mask_box((64, 64), 100) == (0, 0, 0)      # l = 0
    assert img._mask_box((64, 64), -5) == (0, 0, 0)       # l < 0: empty slices
    assert img._mask_box((64, 40), 10) == (26, 26, 6)     # the box ends at column 38
    for shape, r in (((64, 40), 4), ((64, 64), 1.5), ((128, 40), 10)):
        with pytest.raises(ValueError):
            img._mask_box(shape, r)


def test_working_set_beyond_free_memory_raises(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device work after the memory check")
    monkeypatch.setattr(ops, "fft2_mask", fail)
    monkeypatch.setattr(ops, "fft2_sub", fail)
    monkeypatch.setattr(torch.Tensor, "to", fail)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 1 << 30))
    with pytest.raises(MemoryError):
        utils.FFTmask(np.zeros((256, 256), np.float32))
    with pytest.raises(MemoryError):
        utils.FFTsub(np.zeros((256, 256)), np.zeros((256, 256), np.complex64))


def test_threshimg_on_the_host():
    d = np.array([[0.1, 0.25, 0.5], [0.75, 0.9, np.nan]])
    want = np.array([[True, False, False], [False, True, False]])
    assert np.array_equal(utils.threshImg(d), want) and utils.threshImg(d).dtype == bool
    t = utils.threshImg(torch.from_numpy(d), 0.3, 0.6)
    assert t.dtype == torch.bool and np.array_equal(t.numpy(), fft_ref.threshimg(d, 0.3, 0.6))


def test_signatures_equal_the_reference():
    ref = {
        "FFTmask": "(imgsrc, maskratio=10)",
        "FFTsub": "(imgsrc, imgfft)",
        "threshImg": "(diff, threshL=0.25, threshH=0.75)",
    }
    for name, sig in ref.items():
        f = getattr(utils, name)
        assert f is getattr(img, name)
        s = inspect.signature(f)
        plain = s.replace(parameters=[p.replace(annotation=p.empty) for p in s.parameters.values()],
                          return_annotation=s.empty)
        assert str(plain) == sig, name
