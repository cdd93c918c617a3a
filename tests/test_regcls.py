"""Regressor / Classifier without a GPU: the float64 oracle against the reference goldens, the
module tree and state_dict against the reference's, argument errors, data preprocessing and the
unchanged `select_loss('nll')`."""
from collections import OrderedDict

import numpy as np
import pytest
import torch

import golden_utils as gu
from atomai_b200.nets import ClassifierNet, RegressorNet, init_cls_model, init_reg_model
from oracle import regcls_ref
from regcls_cases import CASES, inputs, sampled, weights


def rel(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(a - ref).max() / (np.abs(ref).max() + 1e-30))


def _net(c):
    return (RegressorNet if c["kind"] == "reg" else ClassifierNet)(c["ic"], c["out"], "mobilenet")


@pytest.mark.parametrize("name", list(CASES))
def test_keys_and_shapes_match_reference(name):
    c = CASES[name]
    gold = gu.load(f"regcls_{name}.npz")
    sd = _net(c).state_dict()
    assert list(sd) == list(gold["keys"])
    assert [str(tuple(v.shape)) for v in sd.values()] == list(gold["shapes"])


@pytest.mark.parametrize("name", list(CASES))
def test_float64_oracle_vs_reference(name):
    """The float64 restatement reproduces the reference's fp32 outputs, loss and gradients."""
    c = CASES[name]
    gold = gu.load(f"regcls_{name}.npz")
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in _net(c).state_dict().items())
    sd = {k: torch.from_numpy(v).double() if v.dtype != np.int64 else torch.from_numpy(v)
          for k, v in weights(shapes, c).items()}
    x, y = inputs(c)
    x = torch.from_numpy(x).double()
    y = torch.from_numpy(y).double() if c["kind"] == "reg" else torch.from_numpy(y)
    with torch.no_grad():
        assert rel(regcls_ref.forward(c["kind"], x, sd, False), gold["out_eval"]) < 1e-4
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()
              if v.dtype.is_floating_point and "running_" not in k}
    work = dict(sd)
    work.update(leaves)
    stats = {}
    out = regcls_ref.forward(c["kind"], x, work, True, stats)
    loss = regcls_ref.loss(c["kind"], out, y)
    loss.backward()
    assert rel(out.detach(), gold["out_train"]) < 1e-3
    assert abs(loss.item() - float(gold["loss"])) < 1e-4 * abs(float(gold["loss"])) + 1e-6
    er = rr = 0.0
    for k, p in leaves.items():
        got, ref = sampled(p.grad.numpy()), gold["grad/" + k].astype(np.float64)
        er += float(((got - ref) ** 2).sum())
        rr += float((ref ** 2).sum())
    # reg3_32 ends at 1x1 maps: its last BatchNorms normalise over 8 samples per channel, and the
    # reference's own fp32 gradients sit 2.0e-2 (grel) from float64 there; 2.5e-3 elsewhere
    assert (er / rr) ** 0.5 < (5e-2 if name == "reg3_32" else 1e-2)
    for k, v in stats.items():
        assert rel(sampled(v.numpy()), gold["stat/" + k]) < 1e-4


def test_argument_errors():
    from atomai_b200.models import Classifier
    for bb in ("resnet", "vgg"):
        with pytest.raises(NotImplementedError, match="mobilenet"):
            RegressorNet(1, 2, bb)
        with pytest.raises(NotImplementedError, match="mobilenet"):
            ClassifierNet(1, 2, bb)
    with pytest.raises(AssertionError, match="nb_classes"):
        Classifier()


def test_meta_dicts():
    _, m = init_reg_model(3, "mobilenet", input_channels=2)
    assert m == {"model_type": "reg", "backbone": "mobilenet", "in_channels": 2, "out_dim": 3}
    _, m = init_cls_model(5, "mobilenet")
    assert m == {"model_type": "cls", "backbone": "mobilenet", "in_channels": 1, "nb_classes": 5}


def test_preprocessing():
    from atomai_b200.utils import preprocess_training_cls_data, preprocess_training_reg_data
    X = np.random.rand(10, 16, 16).astype(np.float32)
    with pytest.warns(UserWarning, match="channel dimension"):
        Xtr, ytr, Xte, yte = preprocess_training_reg_data(X, np.arange(10.), X[:4], np.arange(4.), 4)
    assert Xtr[0].shape == (4, 1, 16, 16) and ytr[0].shape == (4, 1) and ytr[0].dtype == torch.float32
    with pytest.raises(TypeError):
        preprocess_training_reg_data(X, torch.zeros(10), X, np.zeros(10), 4)
    with pytest.raises(TypeError, match="int64"):
        preprocess_training_cls_data(X[:, None], np.zeros(10, np.int32), X[:, None],
                                     np.zeros(10, np.int64), 4)
    Xtr, ytr, _, _ = preprocess_training_cls_data(X[:, None], np.zeros(10, np.int64), X[:, None],
                                                  np.zeros(10, np.int64), 5)
    assert Xtr[0].shape == (5, 1, 16, 16) and ytr[0].dtype == torch.int64


def test_output_dimension_check():
    from atomai_b200.trainers import RegTrainer
    t = RegTrainer(out_dim=2)
    t.full_epoch, t.batch_size = False, 4
    X = np.random.rand(12, 1, 16, 16).astype(np.float32)
    with pytest.raises(AssertionError, match="output dimensions"):
        t.set_data(X, np.zeros((12, 3), np.float32), X, np.zeros((12, 3), np.float32))


def test_select_loss_nll_unchanged():
    from atomai_b200.losses_metrics import select_loss
    with pytest.raises(NotImplementedError):
        select_loss("nll")


def test_augmentor_kwargs():
    from atomai_b200.transforms import reg_augmentor
    assert reg_augmentor() is None
    with pytest.raises(NotImplementedError, match="rotation"):
        reg_augmentor(rotation=True)
