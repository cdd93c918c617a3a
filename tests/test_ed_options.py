"""Argument checks of the class-conditioned VAE / rVAE and of ImSpec's 1-D decoder_upsampling:
each error is raised on the host, before any device work (the trainer and the networks are replaced
by stubs that fail if they are reached)."""
import numpy as np
import pytest
import torch

import golden_utils as gu


def _no_device(m, monkeypatch):
    def reached(*a, **k):
        raise AssertionError("device work was reached")
    for name in ("compile_trainer", "encode", "train_epoch"):
        if hasattr(m, name):
            monkeypatch.setattr(m, name, reached)
    for net in ("encoder_net", "decoder_net", "net"):
        if getattr(m, net, None) is not None:
            monkeypatch.setattr(getattr(m, net), "forward", reached)
            if hasattr(getattr(m, net), "decode"):
                monkeypatch.setattr(getattr(m, net), "decode", reached)


@pytest.fixture(params=["vae", "rvae"])
def model(request, monkeypatch):
    from atomai_b200.models import VAE, rVAE

    def make(nb_classes):
        m = (VAE if request.param == "vae" else rVAE)((16, 16), latent_dim=2, nb_classes=nb_classes)
        _no_device(m, monkeypatch)
        return m
    return make


X = gu.images(1, 6, 16, 16)


def test_labels_without_classes(model):
    with pytest.raises(RuntimeError, match="forgotten to specify number of classes"):
        model(0).fit(X, np.array([0, 1, 2, 0, 1, 2]))


@pytest.mark.parametrize("y_train, y_test", [([0, 1, 1, 0, 1, 0], None),
                                             ([0, 1, 2, 0, 1, 2], [0, 1, 0, 1, 0, 1])])
def test_class_count_mismatch(model, y_train, y_test):
    m = model(3)
    with pytest.raises(RuntimeError, match="number of classes specified at initialization"):
        m.fit(X, np.array(y_train), None if y_test is None else X, None if y_test is None else np.array(y_test))


def test_label_out_of_range(model):
    with pytest.raises(AssertionError, match="maximum label value must be less than"):
        model(3).fit(X, np.array([0, 1, 3, 0, 1, 3]))
    with pytest.raises(AssertionError, match="maximum label value must be less than"):
        model(3).fit(X, np.array([0, 1, 2, 0, 1, 2]), X, torch.tensor([0, 1, 5, 0, 1, 5]))


@pytest.mark.parametrize("y", [np.array([-1, 0, 1, -1, 0, 1]), np.array([0, 0.5, 1, 0, 0.5, 1]),
                               np.array([0, 1, np.nan, 0, 1, np.nan]), np.array(["a", "b", "c"] * 2)])
def test_negative_or_non_integral_labels(model, y):
    with pytest.raises(ValueError, match="class labels must be"):
        model(3).fit(X, y)


def test_conditional_fit_needs_labels(model):
    with pytest.raises(ValueError, match="nb_classes=3"):
        model(3).fit(X)
    with pytest.raises(ValueError, match="nb_classes=3"):
        model(3).fit(X, np.array([0, 1, 2, 0, 1, 2]), X)


def test_decode_and_reconstruct_arguments(model):
    m = model(3)
    z = np.zeros((4, 2), np.float32)
    with pytest.raises(ValueError, match="nb_classes=3"):
        m.decode(z)
    with pytest.raises(AssertionError, match="maximum label value"):
        m.decode(z, 3)
    with pytest.raises(ValueError, match="non-negative"):
        m.decode(z, np.array(-1))
    with pytest.raises(ValueError, match="2 labels for 4 latent vectors"):
        m.decode(z, torch.tensor([0, 1]))
    with pytest.raises(ValueError, match="nb_classes=3"):
        m.reconstruct(X)
    with pytest.raises(AssertionError, match="maximum label value"):
        m.reconstruct(X, label=7)
    with pytest.raises(AssertionError, match="maximum label value"):
        model(0).decode(z, 0)


def test_host_labels_cast():
    from atomai_b200.models.dgm.vae import host_labels
    y = host_labels(torch.tensor([0., 2., 1.]), 3)
    assert y.dtype == np.int64 and y.tolist() == [0, 2, 1]
    assert host_labels(2, 3).tolist() == [2]


@pytest.mark.parametrize("out_dim", [(30,), (31,)])
def test_imspec_upsampling_length(monkeypatch, out_dim):
    from atomai_b200.models import ImSpec
    m = ImSpec((16, 16), out_dim, 4, decoder_upsampling=True)
    _no_device(m, monkeypatch)
    X, Y = gu.images(2, 4, 16, 16), np.zeros((4, *out_dim), np.float32)
    with pytest.raises(ValueError, match="multiple of 4"):
        m.fit(X, Y, X, Y, training_cycles=1)
    with pytest.raises(ValueError, match="multiple of 4"):
        m.predict(X)


def test_imspec_upsampling_constructor_is_permissive():
    """As in the reference, the constructor accepts any length (fc sized for length // 4)."""
    from atomai_b200.nets import init_imspec_model
    net, _ = init_imspec_model((16, 16), (30,), 4, decoder_upsampling=True, nbfilters_decoder=8)
    assert net.decoder.fc.out_features == 8 * 7


def test_avgpool_refuses_gradient_input():
    from atomai_b200.engine import Act, Tape
    tape = Tape(True, True)
    with pytest.raises(NotImplementedError, match="gradient"):
        tape.avgpool(Act(torch.zeros(1, 4, 4, 1), needs_grad=True), 2, 2)


def test_joint_vaes_still_drop_classes():
    from atomai_b200.models import jVAE
    m = jVAE((16, 16), latent_dim=2, discrete_dim=[3], nb_classes=3)
    with pytest.raises(NotImplementedError):
        m.fit(X, np.array([0, 1, 2, 0, 1, 2]))
