"""Regressor / Classifier (MobileNetV2 backbone) on the GPU: the mobilenet.cu kernels against
float64, parity with the reference goldens (tests/golden/regcls_*.npz) in every math mode, a
training step with torch's convolution, BatchNorm, pooling, linear and loss functions patched to
raise, reproducibility, and fit / save / load_model / predict.

Bounds, from values measured on one H100 80GB HBM3 (700 W) against the reference's fp32 CPU
goldens (worst case over the three cases):
  * outputs / loss / running statistics: fp32 7.6e-5, tf32x3 1.6e-4, tf32 7.2e-2 -> bounds 5e-4
    (fp32, tf32x3) and 0.15 (tf32);
  * gradients (grel over all sampled parameters): fp32 1.6e-2, tf32x3 1.7e-2 -> bound 5e-2.  The
    reference's own fp32 gradients are that far from float64 (2.0e-2 on reg3_32, tests/
    test_regcls.py): the 64x64 and 32x32 cases end at 2x2 and 1x1 maps, where BatchNorm
    normalises over 32 (resp. 8) samples per channel and amplifies rounding, as DAE's
    bn_bilinear_64 does.  Single-pass tf32 measures 0.35-0.63 through the 52 BatchNorm layers and
    is only checked for finite gradients below 1.0: use fp32 or tf32x3 where gradients matter;
  * Adam: the first two losses within 1e-2 (measured 5.9e-3); the third loss is not compared.
    The sampled weights after three steps sit 0.23 / 0.17 / 0.47 (reg_64 / cls_100 / reg3_32)
    of the distance they moved from the golden -> bounds 0.5 / 0.35 / 1.0: the biases of the
    BatchNorms in front of a convolution have an analytic gradient of zero, so their gradients
    are rounding noise that Adam turns into learning-rate-sized steps in either direction;
  * gradients against the float64 restatement, per module: worst 4.7e-3 / 1.05e-2 / 2.1e-2 ->
    bounds 1.5e-2 / 3e-2 / 6e-2.
"""
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import atomai_b200 as ab
import golden_utils as gu
from atomai_b200 import _C, ops
from atomai_b200.losses_metrics import MSELoss, NLLLoss
from atomai_b200.nets import ClassifierNet, RegressorNet
from oracle import regcls_ref
from regcls_cases import ADAM_STEPS, CASES, PREDICT, inputs, sampled, weights

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32x3", "tf32"]
OUT_TOL = {"fp32": 5e-4, "tf32x3": 5e-4, "tf32": 0.15}
GRAD_TOL = {"fp32": 5e-2, "tf32x3": 5e-2, "tf32": 1.0}
GRAD64_TOL = {"reg_64": 1.5e-2, "cls_100": 3e-2, "reg3_32": 6e-2}
ADAM_W_TOL = {"reg_64": 0.5, "cls_100": 0.35, "reg3_32": 1.0}
# measured (gloo, 2 ranks on one H100): step loss 2.2e-6, worst module gradient 3.9e-3, test loss
# 6.9e-3, weights 1.1e-2, running statistics 3.9e-2 after five cycles
DP_TOL = {"step_loss": 1e-5, "grad": 1.5e-2, "test_loss": 3e-2, "weight": 3e-2, "stat": 0.1}


def rel(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(a - ref).max() / (np.abs(ref).max() + 1e-30))


def build(c, dev):
    net = (RegressorNet if c["kind"] == "reg" else ClassifierNet)(c["ic"], c["out"], "mobilenet")
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in net.state_dict().items())
    net.load_state_dict({k: torch.from_numpy(v) for k, v in weights(shapes, c).items()})
    return net.to(dev)


def criterion(c):
    return MSELoss() if c["kind"] == "reg" else NLLLoss()


# ------------------------------------------------------------------ kernels against float64
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("hw", [(7, 9), (8, 6)])
@pytest.mark.parametrize("depthwise,cin,cout", [(True, 40, 40), (True, 96, 96), (False, 3, 32),
                                                (False, 1, 32)])
def test_conv3x3_kernels_vs_float64(cuda, stride, hw, depthwise, cin, cout):
    """Forward (with pending relu6(affine) on load and BN sums), weight gradient and depthwise data
    gradient, input a channel slice (ld > C)."""
    g = torch.Generator().manual_seed(cin * 7 + stride)
    n, (h, w) = 3, hw
    big = torch.randn(n, h, w, cin + 8, generator=g).to(cuda)
    x = big[..., 4:4 + cin]                                   # ld = cin + 8
    scale = (torch.rand(cin, generator=g) * 2 + 0.5).to(cuda)
    shift = (torch.randn(cin, generator=g)).to(cuda)
    wt = torch.randn(cout, 1 if depthwise else cin, 3, 3, generator=g).to(cuda)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    y = torch.empty(n, ho, wo, cout, device=cuda)
    stats = torch.zeros(2 * cout, device=cuda, dtype=torch.float64)
    ops.conv3x3_fwd(x, scale, shift, True, wt, depthwise, y, stride, stats)
    xa = torch.clamp(x.double() * scale.double() + shift.double(), 0, 6).permute(0, 3, 1, 2)
    xa.requires_grad_(True)
    w64 = wt.double().requires_grad_(True)
    ref = F.conv2d(xa, w64, None, stride, 1, 1, cin if depthwise else 1)
    got = y.permute(0, 3, 1, 2).double()
    assert rel(got.cpu(), ref.detach().cpu()) < 1e-5
    s1 = ref.detach().sum((0, 2, 3))
    s2 = (ref.detach() ** 2).sum((0, 2, 3))
    assert rel(stats[:cout].cpu(), s1.cpu()) < 1e-5 and rel(stats[cout:].cpu(), s2.cpu()) < 1e-5
    dy = torch.randn(n, ho, wo, cout, generator=g).to(cuda)
    ref.backward(dy.double().permute(0, 3, 1, 2))
    dw = torch.zeros_like(wt)
    ops.conv3x3_wgrad(dy, x, scale, shift, True, depthwise, dw, stride)
    assert rel(dw.cpu(), w64.grad.cpu()) < 1e-5
    if depthwise:
        dx = torch.empty(n, h, w, cin, device=cuda)
        ops.dw3x3_dgrad(dy, wt, dx, stride)
        assert rel(dx.permute(0, 3, 1, 2).cpu(), xa.grad.cpu()) < 1e-5


def test_head_kernels_vs_float64(cuda):
    g = torch.Generator().manual_seed(3)
    a = torch.randn(5, 3, 3, 64, generator=g).to(cuda)
    sc, sh = (torch.rand(64, generator=g) * 3).to(cuda), (torch.randn(64, generator=g) * 3).to(cuda)
    y = torch.empty(5, 1, 1, 64, device=cuda)
    ops.avgpool_relu6_fwd(a, sc, sh, y)
    ref = torch.clamp(a.double() * sc.double() + sh.double(), 0, 6).mean((1, 2))
    assert rel(y.reshape(5, 64).cpu(), ref.cpu()) < 1e-6
    x = torch.randn(37, 7, generator=g).to(cuda) * 5
    lp = torch.empty_like(x)
    ops.log_softmax_fwd(x, lp)
    assert rel(lp.cpu(), F.log_softmax(x.double(), 1).cpu()) < 1e-6
    t = torch.randint(0, 7, (37,), generator=g).to(cuda)
    loss = torch.empty(1, device=cuda)
    ops.nll_fwd_bwd(lp, t, loss)
    assert abs(loss.item() - F.nll_loss(lp.double(), t).item()) < 1e-5
    dy = torch.randn(37, 7, generator=g).to(cuda)
    dx = torch.empty_like(dy)
    ops.log_softmax_bwd(lp, dy, dx)
    xd = x.double().requires_grad_(True)
    F.log_softmax(xd, 1).backward(dy.double())
    assert rel(dx.cpu(), xd.grad.cpu()) < 1e-5


# ------------------------------------------------------------------ network parity
@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("name", list(CASES))
def test_forward_backward_vs_reference(cuda, name, math):
    c = CASES[name]
    gold = gu.load(f"regcls_{name}.npz")
    x, y = (torch.from_numpy(a).to(cuda) for a in inputs(c))
    ab.set_math(math)
    try:
        net = build(c, cuda)
        assert list(net.state_dict()) == list(gold["keys"])
        net.eval()
        with torch.no_grad():
            e_eval = rel(net(x).cpu(), gold["out_eval"])
        net.train()
        out = net(x)
        loss = criterion(c)(out, y)
        loss.backward()
        e_train = rel(out.detach().cpu(), gold["out_train"])
        e_loss = abs(loss.item() - float(gold["loss"])) / abs(float(gold["loss"]))
        er = rr = 0.0
        for k, p in net.named_parameters():
            got = sampled(p.grad.cpu().numpy()).astype(np.float64)
            ref = gold["grad/" + k].astype(np.float64)
            er += float(((got - ref) ** 2).sum())
            rr += float((ref ** 2).sum())
        e_grad = (er / rr) ** 0.5
        e_stat = max(rel(sampled(v.cpu().numpy()), gold["stat/" + k])
                     for k, v in net.state_dict().items() if "running_" in k)
    finally:
        ab.set_math("tf32x3")
    print(f"{name} {math}: eval {e_eval:.2e} train {e_train:.2e} loss {e_loss:.2e} "
          f"grad {e_grad:.2e} stats {e_stat:.2e}")
    assert e_eval < OUT_TOL[math] and e_train < OUT_TOL[math] and e_loss < OUT_TOL[math]
    assert e_stat < OUT_TOL[math]
    assert e_grad < GRAD_TOL[math]


@pytest.mark.parametrize("name", list(CASES))
def test_adam_steps_vs_reference(cuda, name):
    """Three fp32 Adam steps: the first two losses and the sampled final weights.  The weights are
    compared by their distance to the golden relative to the distance they moved."""
    from atomai_b200.optim import FusedAdam
    c = CASES[name]
    gold = gu.load(f"regcls_{name}.npz")
    x, y = (torch.from_numpy(a).to(cuda) for a in inputs(c))
    ab.set_math("fp32")
    try:
        net = build(c, cuda).train()
        w0 = {k: sampled(p.detach().cpu().numpy()) for k, p in net.named_parameters()}
        opt = FusedAdam(net.parameters(), lr=1e-3)
        losses = []
        for _ in range(ADAM_STEPS):
            opt.zero_grad()
            loss = criterion(c)(net(x), y)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    finally:
        ab.set_math("tf32x3")
    de = dm = 0.0
    for k, p in net.named_parameters():
        got = sampled(p.detach().cpu().numpy()).astype(np.float64)
        ref = gold["adam/" + k].astype(np.float64)
        de += float(((got - ref) ** 2).sum())
        dm += float(((ref - w0[k]) ** 2).sum())
    w_rel = (de / dm) ** 0.5
    print(f"{name}: losses {losses} golden {gold['adam_losses']} weights {w_rel:.2e}")
    np.testing.assert_allclose(losses[:2], gold["adam_losses"][:2], rtol=1e-2)
    assert np.isfinite(losses).all()
    assert w_rel < ADAM_W_TOL[name], w_rel


def _native_and_float64_grads(c, dev):
    net = build(c, dev).train()
    x, y = (torch.from_numpy(a).to(dev) for a in inputs(c))
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()
              if v.dtype.is_floating_point and "running_" not in k}
    work = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    work.update(leaves)
    yd = y.double() if c["kind"] == "reg" else y
    out64 = regcls_ref.forward(c["kind"], x.double(), work, True, {})
    regcls_ref.loss(c["kind"], out64, yd).backward()
    ab.set_math("fp32")
    try:
        out = net(x)
        criterion(c)(out, y).backward()
    finally:
        ab.set_math("tf32x3")
    return net, out, out64, leaves


@pytest.mark.parametrize("name", list(CASES))
def test_gradients_vs_float64_oracle_per_module(cuda, name):
    """Native fp32 train step against the float64 restatement on the same GPU: the output, and
    the gradient of every module on its own (relative L2 error per convolution / BatchNorm /
    Linear), so an error confined to one layer cannot hide in an aggregate."""
    c = CASES[name]
    net, out, out64, leaves = _native_and_float64_grads(c, cuda)
    assert rel(out.detach().cpu(), out64.detach().cpu()) < 1e-4
    # per module (a conv weight, or a BatchNorm's weight and bias together): the bias of a
    # BatchNorm in front of a convolution that feeds another batch-statistics BatchNorm has an
    # analytic gradient of zero, so alone it has no meaningful relative error
    acc = {}
    for k, p in net.named_parameters():
        ref = leaves[k].grad
        m = k.rsplit(".", 1)[0]
        e, r = acc.get(m, (0.0, 0.0))
        acc[m] = (e + float((p.grad.double() - ref).pow(2).sum()), r + float(ref.pow(2).sum()))
    errs = {m: (e / r) ** 0.5 for m, (e, r) in acc.items()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    print(name, "worst per-module gradient errors:", [(k, f"{e:.2e}") for k, e in worst])
    bad = {k: e for k, e in errs.items() if e > GRAD64_TOL[name]}
    assert not bad, bad


# ------------------------------------------------------------------ native path only
def test_training_step_uses_no_torch_kernels(cuda, monkeypatch):
    c = CASES["reg_64"]
    net = build(c, cuda).train()
    x, y = (torch.from_numpy(a).to(cuda) for a in inputs(c))
    for name in ("conv2d", "batch_norm", "relu6", "adaptive_avg_pool2d", "linear", "log_softmax",
                 "nll_loss", "mse_loss"):
        def boom(*a, _n=name, **k):
            raise AssertionError(f"torch F.{_n} called on the native path")
        monkeypatch.setattr(F, name, boom)
    calls = []
    for fn in ("conv_fwd", "conv_wgrad", "conv3x3_fwd", "conv3x3_wgrad", "dw3x3_dgrad"):
        orig = getattr(ops, fn)
        monkeypatch.setattr(ops, fn, lambda *a, _o=orig, _f=fn, **k: (calls.append(_f), _o(*a, **k))[1])
    out = net(x)
    loss = MSELoss()(out, y)
    loss.backward()
    cls = ClassifierNet(1, 4, "mobilenet").to(cuda).train()
    NLLLoss()(cls(x), torch.arange(8, device=cuda) % 4).backward()
    torch.cuda.synchronize()
    assert all(p.grad is not None for p in net.parameters())
    # 52 convolutions: 1 stem + 17 depthwise + 16 expand + 17 project + the 320 -> 1280 layer
    assert calls.count("conv3x3_fwd") == 2 * 18 and calls.count("conv3x3_wgrad") == 2 * 18
    assert calls.count("dw3x3_dgrad") == 2 * 17


def test_fp32_training_is_bit_reproducible(cuda):
    from atomai_b200.optim import FusedAdam
    c = CASES["cls_100"]
    x, y = (torch.from_numpy(a).to(cuda) for a in inputs(c))
    finals = []
    ab.set_math("fp32")
    try:
        for _ in range(2):
            net = build(c, cuda).train()
            opt = FusedAdam(net.parameters(), lr=1e-3)
            for _ in range(3):
                opt.zero_grad()
                NLLLoss()(net(x), y).backward()
                opt.step()
            finals.append({k: v.detach().clone() for k, v in net.state_dict().items()})
    finally:
        ab.set_math("tf32x3")
    for k in finals[0]:
        assert torch.equal(finals[0][k], finals[1][k]), k


# ------------------------------------------------------------------ models
def _data(kind, n=40, hw=32, out=2, seed=0):
    rs = np.random.RandomState(seed)
    X = gu.images(seed, n, hw, hw)
    if kind == "reg":
        y = np.stack([X.mean((1, 2)), X.std((1, 2))], 1).astype(np.float32)[:, :out]
    else:
        y = (np.arange(n) % out).astype(np.int64)
        rs.shuffle(y)
    return X, y


def test_regressor_fit_save_load_predict(cuda, tmp_path):
    from atomai_b200.models import Regressor, load_model
    X, y = _data("reg")
    m = Regressor(out_dim=2)
    m.fit(X, y, training_cycles=4, batch_size=4, filename=str(tmp_path / "reg"),
          plot_training_history=False)
    assert len(m.loss_acc["train_loss"]) == 4 and np.isfinite(m.loss_acc["train_loss"]).all()
    p = m.predict(X[:5], verbose=False)
    assert p.shape == (5, 2)
    m2 = load_model(str(tmp_path / "reg_metadict_final.tar"))
    np.testing.assert_array_equal(m2.predict(X[:5], verbose=False), p)
    with pytest.raises(AssertionError):
        Regressor(out_dim=3).fit(X, y, training_cycles=1, batch_size=4,
                                 filename=str(tmp_path / "bad"))


def test_classifier_fit_save_load_predict(cuda, tmp_path):
    from atomai_b200.models import Classifier, load_model
    X, y = _data("cls", out=3)
    m = Classifier(nb_classes=3)
    m.fit(X, y, training_cycles=3, batch_size=4, full_epoch=True, compute_accuracy=True,
          filename=str(tmp_path / "cls"), plot_training_history=False)
    assert len(m.loss_acc["train_accuracy"]) == 3
    p = m.predict(X[:7], verbose=False)
    assert p.shape == (7,) and p.dtype == np.int64 and ((0 <= p) & (p < 3)).all()
    m2 = load_model(str(tmp_path / "cls_metadict_final.tar"))
    np.testing.assert_array_equal(m2.predict(X[:7], verbose=False), p)


def test_reference_format_checkpoints_predict_golden(cuda, tmp_path):
    """A checkpoint written the way the reference writes it ('reg' / 'cls' meta dict, case
    weights) loads through load_model and predicts the reference's outputs."""
    from atomai_b200.models import load_model
    gold = gu.load("regcls_load.npz")
    imgs = gold["images"]
    for name in ("reg_64", "cls_100"):
        c = CASES[name]
        net = build(c, "cpu")
        meta = dict(eval(str(gold[f"{name}/meta"])))
        meta["weights"] = net.state_dict()
        meta["optimizer"] = torch.optim.Adam(net.parameters(), lr=1e-3)
        torch.save(meta, str(tmp_path / f"{name}.tar"))
        model = load_model(str(tmp_path / f"{name}.tar"))
        for norm in (True, False):
            got = model.predict(imgs, norm=norm, verbose=False)
            ref = gold[f"{name}/predict_norm{int(norm)}"]
            if c["kind"] == "reg":
                assert rel(got, ref) < 1e-4, (name, norm)
            else:
                np.testing.assert_array_equal(got, ref)


# ------------------------------------------------------------------ data parallelism
def _run_dp(extra, port):
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                        "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port",
                        str(port), os.path.join(root, "tools", "dp_regcls.py")] + extra,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    outs = [json.loads(l) for l in r.stdout.splitlines() if l.startswith("{")]
    assert sorted(o["model"] for o in outs) == ["cls", "reg"], r.stdout[-2000:]
    for o in outs:
        print(o)
        assert o["world"] == 2
        # SyncBN makes the sharded step the global-batch step up to summation order
        assert o["step_loss_rel"] <= DP_TOL["step_loss"] and o["grad_rel"] <= DP_TOL["grad"], o
        assert o["first_loss_rel"] <= DP_TOL["step_loss"], o
        # over five Adam steps that order becomes small weight differences, which this network's
        # 2x2 BatchNorms amplify (see test_adam_steps_vs_reference)
        assert o["test_loss_rel"] <= DP_TOL["test_loss"] and o["weight_rel"] <= DP_TOL["weight"], o
        assert o["stat_rel"] <= DP_TOL["stat"], o


def test_two_rank_fit_equals_single_process(cuda):
    """Regressor / Classifier fit on 2 GPUs (NCCL, SyncBN over NVLink) == one process at the
    global batch."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_dp([], 29745)


def test_two_rank_fit_on_one_gpu_gloo(cuda):
    """The same comparison with two ranks sharing one GPU over gloo: it runs the SyncBN count /
    statistics all-reduce, the per-block BatchNorm finalise and the global backward sums of the
    MobileNet layers wherever a single GPU is available."""
    _run_dp(["--backend", "gloo"], 29746)


def test_out_of_range_labels_raise(cuda):
    from atomai_b200.models import Classifier
    X = gu.images(5, 12, 32, 32)
    y = (np.arange(12) % 3 + 1).astype(np.int64)           # 1-based labels for nb_classes=3
    with pytest.raises(ValueError, match=r"\[0, 2\]"):
        Classifier(nb_classes=3).fit(X, y, X, y, training_cycles=1, batch_size=4,
                                     plot_training_history=False)
