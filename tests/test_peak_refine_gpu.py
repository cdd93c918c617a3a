"""Peak refinement on the GPU (atomai_b200_peak_refine, MINPACK lmdif in fp64, one warp per atom)
against noise-free Gaussians, the scipy oracle and the unmodified reference's goldens
(tests/golden/peak_refine.npz).  The fits are bitwise equal to the reference only up to rounding:
CUDA's exp / sin / cos and the warp reductions round differently from the CPU, and ill-posed fits
(theta free while sigma_x = sigma_y, fits that reach maxfev) amplify that.  The bounds: the
keep/refine decision agrees on >= 99.75 % of atoms (one flip is allowed in sets under 800
atoms), and of the atoms refined by both, >= 99.75 %
agree within 1e-3 px and >= 95 % within 1e-6 px."""
import warnings

import numpy as np
import pytest
import torch

import golden_utils as gu
import refine_cases as rc
from atomai_b200.utils import coords
from oracle import refine_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return gu.load("peak_refine.npz")


def _quiet(fn, *a, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **kw)


def check_parity(got, want, unrefined, label):
    assert got.shape == want.shape
    assert np.array_equal(got[:, 2], want[:, 2])
    moved_g = (got[:, :2] != unrefined[:, :2]).any(1)
    moved_w = (want[:, :2] != unrefined[:, :2]).any(1)
    n = len(want)
    flips = int((moved_g != moved_w).sum())
    both = moved_g & moved_w
    err = np.abs(got[both, :2] - want[both, :2]).max(1)
    n3, n6 = int((err <= 1e-3).sum()), int((err <= 1e-6).sum())
    print(f"{label}: {n} atoms, decision flips {flips}, refined by both {int(both.sum())}: "
          f"{n3} within 1e-3 px, {n6} within 1e-6 px, max {err.max() if len(err) else 0:.2e}")
    assert flips <= max(1, int(0.0025 * n))   # 6 of 2410; one for the 376-atom Locator stack
    assert n3 >= 0.9975 * both.sum() and n6 >= 0.95 * both.sum()


def test_noise_free_gaussians(cuda):
    """Separated Gaussians with known parameters: centres to 1e-6 px, the oracle to 1e-9 px."""
    rs = np.random.RandomState(5)
    H = W = 256
    d = 5
    img = np.full((H, W), 0.1)
    xs, ys = np.mgrid[:H, :W].astype(np.float64)
    truth = []
    for cx in range(16, H - 16, 28):
        for cy in range(16, W - 16, 28):
            x0, y0 = cx + rs.uniform(-0.45, 0.45), cy + rs.uniform(-0.45, 0.45)
            sx, sy, th = rs.uniform(1.1, 1.6), rs.uniform(1.1, 1.6), rs.uniform(-0.6, 0.6)
            win = (slice(cx - 12, cx + 12), slice(cy - 12, cy + 12))
            img[win] += ref.gaussian_2d((xs[win] - x0, ys[win] - y0), 1.0, 0, 0, sx, sy, th,
                                        0).reshape(24, 24)
            truth.append((cx, cy, x0, y0))
    img = img.astype(np.float32)
    truth = np.array(truth)
    xy = np.concatenate([truth[:, :2], np.zeros((len(truth), 1))], 1)
    got = coords.peak_refinement(img, xy, d)
    assert np.abs(got[:, :2] - truth[:, 2:]).max() < 1e-6
    want = ref.peak_refinement(img, xy, d)
    assert np.abs(got - want).max() < 1e-9


@pytest.mark.parametrize("d", [None, 6])
def test_golden_frame(cuda, gold, d):
    frame, xy = rc.bfo_frame()
    got = _quiet(coords.peak_refinement, frame, xy, d)
    check_parity(got, gold[f"bfo_d{d}"], xy, f"bfo d={d}")
    # a CUDA tensor input gives the same result
    got_t = _quiet(coords.peak_refinement, torch.from_numpy(frame).to(cuda), xy, d)
    assert np.array_equal(got_t, got)


def test_locator_golden(cuda, gold, capsys):
    from atomai_b200.predictors import Locator
    nn_out, stack = rc.locator_inputs()
    with pytest.warns(UserWarning, match="Defaulting to 1/4"):
        loc = Locator(refine=True).run(nn_out, stack)
    out = capsys.readouterr().out
    assert "Refining atomic positions... " in out and "Done" in out
    assert list(loc.keys()) == list(gold["loc_keys"])
    for k in loc:
        assert loc[k].shape == gold[f"loc_{k}"].shape
    cat = [np.concatenate([v[k] for k in loc]) for v in
           (loc, {k: gold[f"loc_{k}"] for k in loc}, {k: gold[f"loc_{k}_coords"] for k in loc})]
    check_parity(*cat, "locator, all frames")
    with pytest.raises(AssertionError, match="Pass input image"):
        Locator(refine=True).run(nn_out)


def test_segmentor_predict_refine_end_to_end(cuda, gold):
    """pretrained/bfo weights on the golden 1024^2 image, fp32 math: the atoms whose unrefined
    coordinates equal the golden's meet the parity bounds."""
    import atomai_b200 as ab
    from atomai_b200.models import Segmentor
    ab.set_math("fp32")
    w = gu.load("bfo_weights.npz")
    g = gu.load("bfo_1024.npz")
    m = Segmentor("Unet", nb_classes=3)
    m.net.load_state_dict({k: torch.from_numpy(w[k]) for k in w.files})
    _, plain = m.predict(g["image"], verbose=False)
    _, refined = _quiet(m.predict, g["image"], refine=True, d=4, verbose=False)
    same = (plain[0] == g["coordinates"]).all(1)
    assert same.mean() > 0.99
    check_parity(refined[0][same], gold["bfo_dNone"][same], g["coordinates"][same], "predict")
    _, refined2 = _quiet(m.predict, g["image"], refine=True, d=4, verbose=False)
    assert np.array_equal(refined[0], refined2[0])


def test_reproducible_and_edge_cases(cuda, gold):
    frame, xy = rc.bfo_frame()
    a = coords.peak_refinement(frame, xy[:500], 4)
    b = coords.peak_refinement(frame, xy[:500], 4)
    assert np.array_equal(a, b)
    assert coords.peak_refinement(frame, np.empty((0, 3)), 4).shape == (0, 3)
    for d in (0, 17):
        with pytest.raises(ValueError, match="1 <= d <= 16"):
            coords.peak_refinement(frame, xy[:5], d)
    bad = frame.copy()
    c = np.around(xy[7, :2]).astype(int)
    bad[c[0], c[1]] = np.nan
    with pytest.raises(ValueError):
        coords.peak_refinement(bad, xy[:20], 4)
    # refine=False output is unchanged
    from atomai_b200.predictors import Locator
    nn_out, stack = rc.locator_inputs()
    plain = Locator(refine=False).run(nn_out, stack)
    for k in plain:
        assert np.array_equal(plain[k], gold[f"loc_{k}_coords"])
