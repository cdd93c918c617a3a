"""FFTmask / FFTsub / threshImg on the GPU: every golden case through numpy and CUDA inputs
matches the reference (dtype, shape, errors, mask zeros exactly, values within the bounds of
tests/golden/fft_cases.py); large power-of-two, Bluestein and non-square images match the float64
host restatement (oracle/fft_ref.py); threshImg of the GPU's own difference equals numpy's;
repeated calls give identical bits."""
import os

import numpy as np
import pytest
import torch

import fft_cases as fc
from atomai_b200 import utils
from oracle import fft_ref

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda")]

GOLD = fc.load_golden(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                    "fft_ref.npz"))
CASES = fc.all_cases()


def gold(key):
    return GOLD[key]


def _cuda_fns():
    def wrap(f):
        def g(*a, **k):
            return f(*[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a], **k)
        return g
    return {n: wrap(getattr(utils, n)) for n in ("FFTmask", "FFTsub", "threshImg")}


def _check(name, fns, cuda_out):
    import builtins
    from test_fft import check_against_gold
    if f"{name}/error" in GOLD.files:
        with pytest.raises(getattr(builtins, str(GOLD[f"{name}/error"]))):
            fc.call(fns, name, gold)
        return
    got = fc.call(fns, name, gold)
    got = got if isinstance(got, tuple) else (got,)
    if cuda_out:
        assert all(isinstance(g, torch.Tensor) and g.is_cuda for g in got)
        got = tuple(g.cpu().numpy() for g in got)
    check_against_gold(name, got)


@pytest.mark.parametrize("name", list(CASES))
def test_goldens_numpy_inputs(name):
    _check(name, utils, False)


@pytest.mark.parametrize("name", list(CASES))
def test_goldens_cuda_inputs(name):
    _check(name, _cuda_fns(), True)


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("thresh_")])
def test_threshimg_golden_bounds(name):
    """threshImg of the GPU's own FFTsub against the reference's, except pixels whose reference
    difference lies within the FFTsub bound of a threshold"""
    _, args, kw = CASES[name]
    src_case = name.split("_")[1] + "_" + name.split("_")[2]
    src, spec = CASES[src_case][1](gold)
    ref_d = GOLD[f"{src_case}/out"]
    d = utils.FFTsub(src, spec)
    _, raw = fft_ref.fftsub(src, spec, raw=True)
    tol = fc.sub_tol(src, spec, raw, spec.dtype == np.complex64)
    lo, hi = kw.get("threshL", 0.25), kw.get("threshH", 0.75)
    exempt = (np.abs(ref_d - lo) <= tol) | (np.abs(ref_d - hi) <= tol)
    got, want = utils.threshImg(d, **kw), GOLD[f"{name}/out"]
    assert got.dtype == want.dtype == bool
    assert np.array_equal(got[~exempt], want[~exempt])
    assert np.array_equal(got, fft_ref.threshimg(d, lo, hi))


def _image(h, w, dtype=np.float64):
    return fc.image(h, w, h + 7 * w, dtype)


LARGE = [(256, 256), (1024, 1024), (4096, 4096), (8192, 8192), (1000, 1000), (4093, 4093),
         (4096, 1000), (3000, 4096)]


@pytest.mark.parametrize("h, w", LARGE, ids=[f"{h}x{w}" for h, w in LARGE])
def test_float64_against_oracle(h, w):
    x = _image(h, w)
    # a 4096 x 1000 image is narrower than the default disk's box (ValueError, as in the
    # reference); a negative ratio masks nothing
    r = 10 if w >= h // 2 + h // 10 else -5
    R2, R3 = fft_ref.fftmask(x, r)
    F2, F3 = utils.FFTmask(torch.from_numpy(x).cuda(), r)
    assert F2.dtype == F3.dtype == torch.complex128
    F2, F3 = F2.cpu().numpy(), F3.cpu().numpy()
    tol = fc.spectrum_tol(R2, False)
    assert np.linalg.norm(F2 - R2) <= tol and np.linalg.norm(F3 - R3) <= tol
    assert np.array_equal(fc.masked(F2, F3), fc.masked(R2, R3))
    del F2, R2
    # zero the low frequencies, so the difference is well above rounding noise
    F3[h // 2 - h // 20:h // 2 + h // 20, w // 2 - w // 20:w // 2 + w // 20] = 0
    d = utils.FFTsub(torch.from_numpy(x).cuda(), torch.from_numpy(F3).cuda())
    ref, raw = fft_ref.fftsub(x, F3, raw=True)
    stol = fc.sub_tol(x, F3, raw, False)
    assert d.dtype == torch.float64 and stol is not None
    dn = d.cpu().numpy()
    assert np.abs(dn - ref).max() <= stol
    t = utils.threshImg(d)
    assert t.dtype == torch.bool and np.array_equal(t.cpu().numpy(), fft_ref.threshimg(dn))


@pytest.mark.parametrize("h, w", fc.SIZES, ids=[f"{h}x{w}" for h, w in fc.SIZES])
def test_float64_golden_sizes_against_oracle(h, w):
    """the float64 path at every golden size (the size goldens themselves are float32)"""
    x = _image(h, w)
    r = 10 if w >= h // 2 + h // 10 else -5
    R2, R3 = fft_ref.fftmask(x, r)
    F2, F3 = utils.FFTmask(x, r)
    assert F2.dtype == F3.dtype == np.complex128 and F2.shape == (h, w)
    tol = fc.spectrum_tol(R2, False)
    assert np.linalg.norm(F2 - R2) <= tol and np.linalg.norm(F3 - R3) <= tol
    assert np.array_equal(fc.masked(F2, F3), fc.masked(R2, R3))
    spec = R2.copy()
    spec[h // 2 - h // 8:h // 2 + h // 8 + 1, w // 2 - w // 8:w // 2 + w // 8 + 1] = 0
    d = utils.FFTsub(x, spec)
    ref, raw = fft_ref.fftsub(x, spec, raw=True)
    stol = fc.sub_tol(x, spec, raw, False)
    assert d.dtype == np.float64 and d.shape == (h, w)
    if stol is None:   # a 1 x 1 image: one pixel, 0 / 0
        assert np.isnan(d).all() or (np.isfinite(d).all() and d.min() >= 0 and d.max() <= 1)
    else:
        assert np.abs(d - ref).max() <= stol


@pytest.mark.parametrize("h, w", [(1024, 1024), (4093, 4093), (3000, 4096)])
def test_complex64_is_the_rounded_oracle(h, w):
    """float32 input: the float64 result rounded once, within the float64 bound plus one
    complex64 ulp per component"""
    x = _image(h, w, np.float32)
    R2, R3 = fft_ref.fftmask(x.astype(np.float64), 10)
    F2, F3 = utils.FFTmask(x, 10)
    assert F2.dtype == F3.dtype == np.complex64
    tol = fc.spectrum_tol(R2, False)
    for g, r in ((F2, R2), (F3, R3)):
        r32 = r.astype(np.complex64)
        for part in (np.real, np.imag):
            ulp = np.spacing(np.abs(part(r32)))
            assert (np.abs(part(g).astype(np.float64) - part(r32)) <= tol + ulp).all()
    d = utils.FFTsub(x, F3)
    assert d.dtype == np.float32 and d.shape == (h, w)


def test_unmasked_spectrum_gives_bounded_noise():
    x = _image(1000, 1000)
    F2, _ = utils.FFTmask(x)
    d = utils.FFTsub(x, F2)
    assert d.shape == x.shape and d.dtype == np.float64
    assert np.isfinite(d).all() and d.min() >= 0 and d.max() <= 1


def test_constant_difference_is_nan():
    d = utils.FFTsub(np.full((100, 60), 2.5), np.zeros((100, 60), np.complex64))
    assert d.dtype == np.float64 and np.isnan(d).all()


@pytest.mark.parametrize("h, w", [(1000, 1000), (4096, 4096), (97, 8192)])
def test_repeat_calls_identical(h, w):
    x = torch.from_numpy(_image(h, w, np.float32)).cuda()
    a2, a3 = utils.FFTmask(x, 4)
    b2, b3 = utils.FFTmask(x, 4)
    assert torch.equal(a2, b2) and torch.equal(a3, b3)
    assert torch.equal(utils.FFTsub(x, a3), utils.FFTsub(x, a3))
