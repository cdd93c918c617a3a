"""DenoisingAutoencoder without a GPU: the oracle (oracle/dae_ref.py) against goldens produced by
the unmodified reference (tests/golden/make_golden_dae.py), module tree and state_dict keys,
meta_state_dict, checkpoint loading, the data checks of preprocess_denoiser_data, the input-size
check and the refusal to train without CUDA."""
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

import golden_utils as gu
from dae_cases import ADAM_STEPS, CKPT, DAE_CASES, inputs, sampled
from oracle import dae_ref


def build_dae(name):
    """(model [atomai_b200, on the default device], seeded state_dict, cfg, noisy x, clean y,
    golden).  x and y are CPU float32 (n, 1, h, w) tensors."""
    from atomai_b200.models import DenoisingAutoencoder
    c = DAE_CASES[name]
    m = DenoisingAutoencoder(**c["kw"])
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in m.net.state_dict().items())
    sd = OrderedDict((k, torch.from_numpy(v)) for k, v in gu.fill_state_dict(shapes, c["seed"]).items())
    m.net.load_state_dict(sd)
    x, y = (torch.from_numpy(a) for a in inputs(c))
    return m, sd, dict(c["kw"]), x, y, gu.load(f"dae_{name}.npz")


def _f64(sd):
    return OrderedDict((k, v.double() if v.dtype.is_floating_point else v.clone()) for k, v in sd.items())


@pytest.mark.parametrize("name", list(DAE_CASES))
def test_dae_oracle_matches_reference(name):
    _, sd, cfg, x, y, gold = build_dae(name)
    sd, x, y = _f64(sd), x.double(), y.double()
    with torch.no_grad():
        oe = dae_ref.dae_forward(x, sd, cfg, training=False)
    scale = np.abs(gold["out_eval"]).max()
    # measured (float64 oracle vs the reference's fp32): outputs <= 5.5e-6 relative, loss 7e-7,
    # gradients 2e-5 of their norm (bn_bilinear_64; the cases without BatchNorm ~1e-6)
    assert np.abs(oe.numpy() - gold["out_eval"]).max() <= 1e-5 * scale
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()
              if v.dtype.is_floating_point and "running_" not in k}
    work = dict(sd)
    work.update(leaves)
    stats = {}
    ot = dae_ref.dae_forward(x, work, cfg, training=True, new_stats=stats)
    assert np.abs(ot.detach().numpy() - gold["out_train"]).max() <= 1e-5 * np.abs(gold["out_train"]).max()
    loss = torch.nn.functional.mse_loss(ot, y)
    assert abs(loss.item() - float(gold["loss_train"])) <= 1e-5 * float(gold["loss_train"])
    loss.backward()
    for k, p in leaves.items():
        g = sampled(p.grad.numpy())
        gn = float(gold["gradnorm/" + k])
        assert abs(np.linalg.norm(p.grad.numpy()) - gn) <= 1e-4 * gn, k
        assert np.abs(g.reshape(-1) - gold["grad/" + k].reshape(-1)).max() <= 1e-4 * gn + 1e-9, k
    assert set(stats) == {k[len("buf/"):] for k in gold.files if k.startswith("buf/")}
    for k, v in stats.items():
        np.testing.assert_allclose(v.numpy(), gold["buf/" + k], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", list(DAE_CASES))
def test_dae_oracle_adam_steps_match_reference(name):
    _, sd, cfg, x, y, gold = build_dae(name)
    sd = OrderedDict((k, v.clone()) for k, v in sd.items())
    state = {}
    losses = [dae_ref.dae_train_step(x, y, sd, cfg, state)[0] for _ in range(ADAM_STEPS)]
    # With BatchNorm on 4 x 8 x 8 bottleneck samples per channel the trajectory is ill-conditioned:
    # the same fp32 expressions land 1.7e-4 (losses) / 2.4e-4 (weights) from the reference after
    # five steps; without BatchNorm 1e-7.
    bn = cfg.get("use_batch_norm", False)
    np.testing.assert_allclose(losses, gold["adam_losses"], rtol=1e-3 if bn else 2e-5)
    for k in sd:
        if "adam/" + k in gold.files:
            np.testing.assert_allclose(sampled(sd[k].numpy()), gold["adam/" + k],
                                       atol=1e-3 if bn else 2e-5, err_msg=k)


@pytest.mark.parametrize("name", list(DAE_CASES))
def test_module_tree_and_state_dict_keys_match_reference(name):
    from atomai_b200.nets import ConvBlock, DenoisingAutoencoderNet, UpsampleBlock
    m, *_, gold = build_dae(name)
    net = m.net
    assert isinstance(net, DenoisingAutoencoderNet) and isinstance(net, torch.nn.Sequential)
    assert list(net.state_dict()) == list(gold["keys"])
    assert [type(c) for c in net.children()] == [torch.nn.Sequential, torch.nn.Sequential]
    tree = [f"{i}.{j}:{type(c).__name__}" for i, seq in enumerate(net.children())
            for j, c in enumerate(seq.children())]
    assert tree == list(gold["tree"])
    kinds = {"ConvBlock": ConvBlock, "UpsampleBlock": UpsampleBlock,
             "MaxPool2d": torch.nn.MaxPool2d, "Conv2d": torch.nn.Conv2d}
    mods = [c for seq in net.children() for c in seq.children()]
    assert [type(c) for c in mods] == [kinds[t.split(":")[1]] for t in gold["tree"]]
    for k, v in net.state_dict().items():
        if "grad/" + k in gold.files and v.numel() <= 4096:
            assert tuple(v.shape) == gold["grad/" + k].shape, k


def test_meta_state_dict():
    from atomai_b200.models import DenoisingAutoencoder
    m = DenoisingAutoencoder()
    meta = m.meta_state_dict
    assert list(meta) == ["model_type", "encoder_filters", "decoder_filters", "encoder_layers",
                          "decoder_layers", "use_batch_norm", "upsampling_mode", "weights"]
    assert meta["model_type"] == "denoising_autoencoder"
    assert (meta["encoder_filters"], meta["decoder_filters"]) == ([8, 16, 32, 64], [64, 32, 16, 8])
    assert (meta["encoder_layers"], meta["decoder_layers"]) == ([1, 2, 2, 2], [2, 2, 2, 1])
    assert meta["use_batch_norm"] is False and meta["upsampling_mode"] == "nearest"
    assert list(meta["weights"]) == list(m.net.state_dict())
    kw = dict(encoder_filters=[4, 8], decoder_filters=[8, 4], encoder_layers=[1, 1],
              decoder_layers=[1, 1], use_batch_norm=True, upsampling_mode="bilinear")
    m = DenoisingAutoencoder(**kw, seed=3)
    assert all(m.meta_state_dict[k] == v for k, v in kw.items())
    assert m.net.size_multiple == 2 and DenoisingAutoencoder().net.size_multiple == 8
    assert isinstance(m.net[1][1], torch.nn.Module) and m.net[1][1].mode == "bilinear"


def test_same_seed_same_initial_weights():
    from atomai_b200.models import DenoisingAutoencoder
    from atomai_b200.models.denoiser import init_denoising_autoencoder
    a = DenoisingAutoencoder(seed=5).net.state_dict()
    net, meta = init_denoising_autoencoder(seed=5)
    assert meta["model_type"] == "denoising_autoencoder"
    assert all(torch.equal(a[k].cpu(), v.cpu()) for k, v in net.state_dict().items())


def test_load_model_dispatch_and_loader_defaults(tmp_path):
    from atomai_b200.models import DenoisingAutoencoder, load_model
    src = DenoisingAutoencoder(encoder_filters=[8, 16], decoder_filters=[16, 8],
                               encoder_layers=[1, 1], decoder_layers=[1, 1], use_batch_norm=True,
                               upsampling_mode="bilinear")
    full = dict(src.meta_state_dict, weights={k: v.cpu() for k, v in src.net.state_dict().items()})
    torch.save(full, tmp_path / "full.tar")
    m = load_model(str(tmp_path / "full.tar"))
    assert type(m) is DenoisingAutoencoder and not m.net.training
    assert (m.encoder_filters, m.use_batch_norm, m.upsampling_mode) == ([8, 16], True, "bilinear")
    for k, v in src.net.state_dict().items():
        assert torch.equal(m.net.state_dict()[k].cpu(), v.cpu()), k
    # keys missing from a checkpoint take the reference loader's defaults: its use_batch_norm
    # default is True although the class defaults to False
    bare = DenoisingAutoencoder(use_batch_norm=True)
    torch.save({"model_type": "denoising_autoencoder",
                "weights": {k: v.cpu() for k, v in bare.net.state_dict().items()}},
               tmp_path / "bare.tar")
    m = load_model(str(tmp_path / "bare.tar"))
    assert m.use_batch_norm is True and m.meta_state_dict["use_batch_norm"] is True
    assert m.encoder_filters == [8, 16, 32, 64] and m.decoder_layers == [2, 2, 2, 1]
    assert m.upsampling_mode == "nearest"
    assert any(isinstance(c, torch.nn.BatchNorm2d) for c in m.net.modules())


def test_load_reference_checkpoint():
    from atomai_b200.models import DenoisingAutoencoder, load_model
    path = os.path.join(gu.GOLDEN_DIR, "dae_fit.tar")
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert ck["model_type"] == "denoising_autoencoder"
    m = load_model(path)
    assert type(m) is DenoisingAutoencoder
    for k in ("encoder_filters", "decoder_filters", "encoder_layers", "decoder_layers"):
        assert getattr(m, k) == CKPT["kw"][k] == ck[k]
    assert m.use_batch_norm is False and m.upsampling_mode == "nearest"
    sd = m.net.state_dict()
    assert list(sd) == list(ck["weights"])
    for k, v in ck["weights"].items():
        assert torch.equal(sd[k].cpu(), v.cpu()), k
    assert m.optimizer is not None


def test_preprocess_denoiser_data():
    from atomai_b200.utils import preprocess_denoiser_data
    a = np.random.rand(4, 8, 8).astype(np.float64)
    with pytest.warns(UserWarning, match="Adding channel dimension of 1 to noisy training images"):
        out = preprocess_denoiser_data(a, a, a[:2], a[:2])
    assert [tuple(t.shape) for t in out] == [(4, 1, 8, 8)] * 2 + [(2, 1, 8, 8)] * 2
    assert all(isinstance(t, torch.Tensor) and t.dtype == torch.float32 for t in out)
    t4 = torch.rand(4, 1, 8, 8, dtype=torch.float64)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        out = preprocess_denoiser_data(t4, t4, t4[:2], t4[:2])
    assert all(t.dtype == torch.float32 and t.dim() == 4 for t in out)
    with pytest.raises(TypeError):
        preprocess_denoiser_data(a, torch.from_numpy(a), a, a)
    with pytest.raises(ValueError, match="training"):
        preprocess_denoiser_data(a, a[:, :4], a, a)
    with pytest.raises(ValueError, match="test"):
        preprocess_denoiser_data(a, a, a, a[:3])


def test_input_size_must_divide_by_pooling():
    from atomai_b200.models import DenoisingAutoencoder
    m = DenoisingAutoencoder()
    with pytest.raises(ValueError, match="divisible by 8"):
        m.net(torch.zeros(1, 1, 60, 64))
    with pytest.raises(ValueError, match="divisible by 8"):
        m.net(torch.zeros(1, 1, 64, 36))
    with pytest.raises(ValueError, match="divisible by 4"):
        DenoisingAutoencoder(**DAE_CASES["three_level_32"]["kw"]).net(torch.zeros(1, 1, 34, 32))


def test_refuses_to_train_without_cuda(tmp_path):
    from atomai_b200.models import DenoisingAutoencoder
    m = DenoisingAutoencoder()
    m.device = "cpu"
    m.net.cpu()
    x = np.random.rand(8, 16, 16).astype(np.float32)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.fit(x, x, x[:4], x[:4], training_cycles=2, batch_size=4,
              filename=str(tmp_path / "m"), plot_training_history=False)


def test_perturb_weights_refused_with_batch_norm():
    from atomai_b200.models import DenoisingAutoencoder
    x = np.random.rand(8, 1, 16, 16).astype(np.float32)
    with pytest.raises(AssertionError, match="batch normalization"):
        DenoisingAutoencoder(use_batch_norm=True).fit(x, x, x, x, training_cycles=1,
                                                      perturb_weights=True)


def test_exports():
    import atomai_b200.models as models
    import atomai_b200.nets as nets
    import atomai_b200.utils as utils
    for mod, names in ((models, ("DenoisingAutoencoder", "denoise_images")),
                       (nets, ("DenoisingAutoencoderNet",))):
        for n in names:
            assert n in mod.__all__ and hasattr(mod, n), (mod.__name__, n)
    assert hasattr(utils, "preprocess_denoiser_data")
