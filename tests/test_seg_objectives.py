"""CPU checks of the segmentation objectives: the torch restatement (oracle/seg_objectives_ref.py)
against the unmodified reference's outputs (tests/golden/seg_objectives.npz), the reference's
module names, the CUDA-only contract, and the kernels' register budgets."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import golden_utils as gu
import seg_cases as sc
from oracle import seg_objectives_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return gu.load("seg_objectives.npz")


def _grad(fn, x, y):
    xt = torch.from_numpy(x).requires_grad_(True)
    loss = fn(xt, torch.from_numpy(y))
    loss.backward()
    return float(loss.detach()), xt.grad.numpy()


@pytest.mark.parametrize("name", list(sc.CASES))
def test_oracle_dice_matches_reference(gold, name):
    x, y = sc.case(name)
    loss, g = _grad(ref.dice_loss, x, y)
    np.testing.assert_allclose(loss, gold[f"{name}/dice_loss"], rtol=1e-6)
    np.testing.assert_allclose(g, gold[f"{name}/dice_grad"], rtol=1e-6,
                               atol=1e-6 * np.abs(gold[f"{name}/dice_grad"]).max())


def test_dice_reduces_over_batch_and_rows_only():
    """The reference's dims (0, 2) for rank-3 labels: one cell per (class, column), so the loss
    differs from a Dice over whole class maps."""
    x, y = sc.case("mc3_32x48")
    inter, card = ref.dice_cells(torch.from_numpy(x), torch.from_numpy(y))
    assert inter.numel() == 3 * 48
    p = torch.softmax(torch.from_numpy(x), 1)
    t = torch.nn.functional.one_hot(torch.from_numpy(y), 3).permute(0, 3, 1, 2).float()
    whole = 1 - (2 * (p * t).sum((0, 2, 3)) / ((p + t).sum((0, 2, 3)) + 1e-7)).mean()
    assert abs(float(whole) - float(ref.dice_loss(torch.from_numpy(x), torch.from_numpy(y)))) > 1e-3


def test_oracle_focal_matches_reference(gold):
    x, y = sc.case("bin_32x32")
    loss, g = _grad(ref.focal_loss, x, y)
    np.testing.assert_allclose(loss, gold["bin_32x32/focal_loss"], rtol=1e-6)
    np.testing.assert_allclose(g, gold["bin_32x32/focal_grad"], rtol=1e-6,
                               atol=1e-6 * np.abs(gold["bin_32x32/focal_grad"]).max())


@pytest.mark.parametrize("name", list(sc.CASES))
def test_oracle_dice_coefficients_match_autograd(name):
    """dice_finalize's (A, B), chained through the softmax / sigmoid as dice_bwd does, give the
    float64 autograd gradient of the oracle's dice_loss."""
    x, y = sc.case(name)
    x = torch.from_numpy(x).double().requires_grad_(True)
    y = torch.from_numpy(y)
    yy = y.double() if x.shape[1] == 1 else y
    ref.dice_loss(x, yy).backward()
    inter, card = ref.dice_cells(x.detach(), yy)
    A, B = ref.dice_coefficients(inter, card)
    N, C, H, W = x.shape
    if C == 1:
        yl = y[:, 0].long()
        s = torch.sigmoid(x.detach()[:, 0])
        G0 = (yl == 1).double() * A[0] + B[0]
        G1 = (yl == 0).double() * A[1] + B[1]
        g = (s * (1 - s) * (G0 - G1))[:, None]
    else:
        p = torch.softmax(x.detach(), 1)
        t = torch.nn.functional.one_hot(y, C).permute(0, 3, 1, 2).double()
        G = t * A.reshape(1, C, 1, W) + B.reshape(1, C, 1, W)
        g = p * (G - (p * G).sum(1, keepdim=True))
    err = float((g - x.grad).abs().max() / x.grad.abs().max())
    assert err <= 1e-13, err


@pytest.mark.parametrize("gamma", [0.0, 0.5, 1.0, 2.0, 3.7])
@pytest.mark.parametrize("alpha", [0.25, 1.0])
def test_oracle_focal_factor_matches_autograd(alpha, gamma):
    """focal_factor is dfocal/dCE: the oracle's focal_loss gradient over the BCE gradient."""
    for ce in (1e-8, 1e-3, 0.3, 1.0, 7.5, 50.0):
        x = torch.tensor([math.log(math.expm1(ce))], dtype=torch.float64, requires_grad=True)
        t = torch.zeros(1, dtype=torch.float64)
        ref.focal_loss(x, t, alpha, gamma).backward()
        ce64 = torch.nn.functional.binary_cross_entropy_with_logits(x.detach(), t)
        want = float(x.grad) / float(torch.sigmoid(x.detach()))    # dCE/dx = sigmoid(x) at t = 0
        got = float(ref.focal_factor(ce64, alpha, gamma))
        assert abs(got - want) <= 1e-12 * abs(want) + 1e-300, (ce, got, want)
    # CE = 0: autograd's 0 * inf for 0 < gamma < 1 is NaN, and focal_factor says so too
    x = torch.tensor([-1000.0], dtype=torch.float64, requires_grad=True)
    ref.focal_loss(x, torch.zeros(1, dtype=torch.float64), alpha, gamma).backward()
    ce = torch.zeros((), dtype=torch.float64, requires_grad=True)
    (alpha * (1 - torch.exp(-ce)) ** gamma * ce).backward()
    got = ref.focal_factor(torch.zeros((), dtype=torch.float64), alpha, gamma)
    assert torch.equal(got, ce.grad) or (bool(got.isnan()) and bool(ce.grad.isnan()))
    assert bool(x.grad.isnan()) == (0 < gamma < 1)


@pytest.mark.parametrize("name", list(sc.CASES))
def test_oracle_iou_matches_reference(gold, name):
    x, y = sc.case(name)
    counts = ref.iou_counts(torch.from_numpy(y), torch.from_numpy(x))
    assert int(counts.sum()) == y.size
    assert ref.iou_from_counts(counts) == float(gold[f"{name}/iou"])


def test_inputs_keep_away_from_the_threshold():
    for name in sc.CASES:
        x, _ = sc.case(name)
        assert np.abs(sc._probs(x) - 0.5).min() >= sc.MARGIN


def test_reprs_and_select_loss():
    from atomai_b200.losses_metrics import IoU, dice_loss, focal_loss, select_loss
    assert str(select_loss("dice", 3)) == "dice_loss()"
    assert str(select_loss("focal", 1)) == "focal_loss()"
    assert str(dice_loss()) == "dice_loss()" and str(focal_loss()) == "focal_loss()"
    assert callable(IoU)
    with pytest.raises(NotImplementedError):
        focal_loss(with_logits=False)
    with pytest.raises(NotImplementedError, match="dice"):
        select_loss("nll", 3)


def test_cpu_tensors_raise():
    from atomai_b200.losses_metrics import IoU, dice_loss, focal_loss
    x, y = sc.case("mc3_24x37")
    with pytest.raises(RuntimeError):
        dice_loss()(torch.from_numpy(x), torch.from_numpy(y))
    xb, yb = sc.case("bin_32x32")
    with pytest.raises(RuntimeError):
        focal_loss()(torch.from_numpy(xb), torch.from_numpy(yb))
    with pytest.raises(RuntimeError):
        IoU(torch.from_numpy(y), torch.from_numpy(x), 3)


def test_segloss_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-c", "-Xptxas", "-v", os.path.join(ROOT, "atomai_b200", "csrc", "segloss.cu"),
                        "-o", str(tmp_path / "segloss.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    kernels = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    assert len(kernels) == 7, kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) >= len(kernels)
    assert all(a == "0" and b == "0" for a, b in spills), r.stderr
