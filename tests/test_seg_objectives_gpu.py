"""Dice / focal losses and the IoU accuracy on the GPU: against the unmodified reference's goldens
(tests/golden/seg_objectives.npz), against a float64 torch restatement at the benchmark size,
three Adam steps per math mode, the Segmentor.fit call of the reference's segmentation notebook,
bitwise reproducibility and the data-parallel global-batch equivalence."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import golden_utils as gu
import seg_cases as sc
from oracle import seg_objectives_ref as ref
from test_oracle import build_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ["fp32", "tf32", "tf32x3"]
EXACT = ("fp32", "tf32x3")


@pytest.fixture(scope="module")
def gold():
    return gu.load("seg_objectives.npz")


def _loss_grad(crit, x, y):
    xt = x.clone().requires_grad_(True)
    loss = crit(xt, y)
    loss.backward()
    return loss, xt.grad


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


@pytest.mark.parametrize("name", list(sc.CASES))
def test_losses_and_iou_match_reference(cuda, gold, name):
    from atomai_b200.losses_metrics import IoU, dice_loss, focal_loss
    x, y = (torch.from_numpy(a).to(cuda) for a in sc.case(name))
    loss, g = _loss_grad(dice_loss(), x, y)
    assert loss.shape == () and loss.dtype == torch.float32
    assert abs(loss.item() - float(gold[f"{name}/dice_loss"])) <= 1e-5 * abs(float(gold[f"{name}/dice_loss"]))
    assert g.shape == x.shape
    assert _rel(g.cpu(), gold[f"{name}/dice_grad"]) <= 1e-5
    if x.shape[1] == 1:
        loss, g = _loss_grad(focal_loss(), x, y)
        ref_l = float(gold[f"{name}/focal_loss"])
        assert abs(loss.item() - ref_l) <= 1e-5 * abs(ref_l)
        assert _rel(g.cpu(), gold[f"{name}/focal_grad"]) <= 1e-5
    iou = IoU(y, x, x.shape[1])
    assert torch.equal(iou.confusion().cpu(), ref.iou_counts(y.cpu(), x.cpu()))
    v = iou.evaluate()
    assert isinstance(v, float)
    assert abs(v - float(gold[f"{name}/iou"])) <= 1e-7


def _safe_logits(shape, seed, dev):
    """Random logits with no class probability within 1e-4 of the 0.5 threshold."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(shape, device=dev, generator=gen) * 2
    p = torch.sigmoid(x.double()) if shape[1] == 1 else torch.softmax(x.double(), 1)
    bad = ((p - 0.5).abs() < 1e-4).any(1, keepdim=True)
    safe = torch.tensor([3.0] if shape[1] == 1 else [3.0] + [0.0] * (shape[1] - 2) + [-3.0],
                        device=dev).reshape(1, -1, 1, 1)
    return torch.where(bad, safe.expand_as(x), x).contiguous()


@pytest.mark.parametrize("C", [3, 1])
def test_benchmark_size_vs_float64(cuda, C):
    """32 x C x 512^2: many slots of the ordered dice sums, the workspace cap, and exact counts."""
    from atomai_b200.losses_metrics import IoU, dice_loss, focal_loss
    N, H, W = 32, 512, 512
    x = _safe_logits((N, C, H, W), 5, cuda)
    gen = torch.Generator(device=cuda).manual_seed(6)
    if C == 1:
        y = (torch.rand((N, 1, H, W), device=cuda, generator=gen) > 0.5).float()
    else:
        y = torch.randint(0, C, (N, H, W), device=cuda, generator=gen)
    crits = [(dice_loss(), ref.dice_loss)] + ([(focal_loss(), ref.focal_loss)] if C == 1 else [])
    for crit, oracle in crits:
        loss, g = _loss_grad(crit, x, y)
        x64 = x.double().requires_grad_(True)
        l64 = oracle(x64, y.double() if C == 1 else y)
        l64.backward()
        assert abs(loss.item() - l64.item()) <= 1e-5 * abs(l64.item()), (crit, loss.item(), l64.item())
        gd = (g.double() - x64.grad).abs().max() / x64.grad.abs().max()
        assert gd <= 1e-5, (crit, float(gd))
    iou = IoU(y, x, C)
    counts = ref.iou_counts(y, x.double())
    assert torch.equal(iou.confusion(), counts)
    # same counts; torch's GPU mean may differ from the sequential float32 mean in the last bit
    assert abs(iou.evaluate() - ref.iou_from_counts(counts)) <= 1e-7


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("loss", ["dice", "focal"])
def test_three_adam_steps(cuda, gold, loss, math):
    """BaseTrainer.train_step semantics x3 with the fused Adam kernel; losses and the px weights
    at the tolerances of tests/test_unet_gpu.py::test_three_adam_steps.  The first conv layer sits
    behind four BatchNorm backwards over 32x32 (48) images, which turn any last-bit difference
    into ~1e-3 of its gradient (see tests/test_multigpu.py); it gets a norm bound.  The focal loss
    is ~alpha CE^3 at small CE (gamma = 2), so its relative error is three times that of the
    underlying BCE: its loss bound is scaled by 1 + gamma."""
    import atomai_b200 as ab
    from atomai_b200.losses_metrics import select_loss
    from atomai_b200.optim import FusedAdam
    ab.set_math(math)
    net, sd, cfg, x, y, _ = build_case(sc.ADAM[loss])
    net = net.to(cuda)
    x, y = x.to(cuda), y.to(cuda)
    opt = FusedAdam(net.parameters(), lr=1e-3)
    crit = select_loss(loss, cfg["nb_classes"])
    losses = []
    for _ in range(3):
        net.train()
        opt.zero_grad()
        l = crit(net(x), y)
        l.backward()
        opt.step()
        losses.append(l.item())
    ab.set_math("tf32x3")
    np.testing.assert_allclose(losses, gold[f"adam_{loss}/losses"],
                               rtol=(2e-4 if math in EXACT else 3e-3) * (3 if loss == "focal" else 1))
    atol = {"fp32": 2e-5, "tf32x3": 1e-4, "tf32": 1.5e-3}[math]
    np.testing.assert_allclose(net.px.weight.detach().cpu().numpy(), gold[f"adam_{loss}/px_weight"],
                               atol=atol)
    c1 = net.c1.block[0].weight.detach().cpu().double().numpy()
    ref_c1 = gold[f"adam_{loss}/c1_weight"].astype(np.float64)
    r = np.linalg.norm(c1 - ref_c1) / np.linalg.norm(ref_c1)
    assert r <= (5e-3 if math in EXACT else 2e-2), r


def _data(n, h, w, seed):
    return gu.images(seed, n, h, w), gu.labels(seed + 1, n, h, w, 3)


def _fit(tmp_path, tag, T=6, **kw):
    from atomai_b200.models import Segmentor
    X, y = _data(16, 64, 64, 31)
    Xt, yt = _data(8, 64, 64, 33)
    m = Segmentor("Unet", nb_classes=3, seed=1)
    m.fit(X, y, Xt, yt, training_cycles=T, batch_size=8, filename=str(tmp_path / tag),
          plot_training_history=False, **kw)
    return m


def test_notebook_fit_dice_with_accuracy_and_swa(cuda, tmp_path):
    """model.fit(..., loss="dice", compute_accuracy=True, swa=True) of the reference's semantic
    segmentation notebook; deferred read-back gives the same histories."""
    import atomai_b200 as ab
    ab.set_math("tf32x3")
    T = 30      # stochastic weight averaging keeps the last 30 cycles
    m = _fit(tmp_path, "nb", T, loss="dice", compute_accuracy=True, swa=True)
    assert str(m.criterion) == "dice_loss()"
    acc = m.loss_acc
    for k in ("train_accuracy", "test_accuracy", "train_loss", "test_loss"):
        assert len(acc[k]) == T, k
        assert all(isinstance(v, float) for v in acc[k]), k
    assert all(0.0 <= v <= 1.0 for v in acc["train_accuracy"] + acc["test_accuracy"])
    m2 = _fit(tmp_path, "nb2", T, loss="dice", compute_accuracy=True, swa=True, sync_host=False)
    for k in ("train_accuracy", "test_accuracy", "train_loss", "test_loss"):
        assert m2.loss_acc[k] == acc[k], k


def test_dice_training_with_accuracy_is_bitwise_reproducible(cuda, tmp_path):
    import atomai_b200 as ab
    ab.set_math("tf32x3")
    runs = []
    for i in range(2):
        m = _fit(tmp_path, f"rep{i}", 5, loss="dice", compute_accuracy=True)
        runs.append(({k: v.detach().cpu().clone() for k, v in m.net.state_dict().items()},
                     {k: list(v) for k, v in m.loss_acc.items()}))
    (sd0, h0), (sd1, h1) = runs
    assert h0 == h1
    for k in sd0:
        assert torch.equal(sd0[k], sd1[k]), k


def test_two_rank_objectives_equal_single_rank(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                        "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
                        "29733", os.path.join(ROOT, "tools", "dp_seg_objectives.py")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert out["world"] == 2
    assert out["iou_equal"], out
    # tolerances of tests/test_multigpu.py
    assert out["dice_loss_rel"] <= 1e-6 and out["focal_loss_rel"] <= 1e-6, out
    assert out["tail_grad_rel_max"] <= 2e-2 and out["grad_rel"] <= 2e-2, out
    assert out["weight_rel"] <= 2e-2, out
