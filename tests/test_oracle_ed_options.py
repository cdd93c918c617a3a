"""oracle/ed_options_ref.py against goldens of the class-conditioned VAE / rVAE and ImSpec's
encoder_downsampling / 1-D decoder_upsampling, produced by the unmodified reference on the CPU
(tests/golden/make_golden_ed_options.py)."""
from collections import OrderedDict

import numpy as np
import pytest
import torch

import ed_options_cases as cases
import golden_utils as gu
from oracle import ed_options_ref as ref


def _seed(net, seed):
    shapes = OrderedDict((k, tuple(v.shape)) for k, v in net.state_dict().items())
    sd = OrderedDict((k, torch.from_numpy(v)) for k, v in gu.fill_state_dict(shapes, seed).items())
    net.load_state_dict(sd)
    return sd


def build_cvae(tag):
    """(model [atomai_b200, CPU-constructed], enc sd, dec sd, x, labels, eps, golden)."""
    from atomai_b200.models import VAE, rVAE
    c = cases.CVAE_CASES[tag]
    cls = rVAE if c["kind"] == "rvae" else VAE
    m = cls(cases.HW, latent_dim=2, nb_classes=cases.NB_CLASSES, **c["kw"])
    enc = _seed(m.encoder_net, c["seed"])
    dec = _seed(m.decoder_net, c["seed"] + 1)
    x, y, eps = (torch.from_numpy(a) for a in cases.cvae_inputs(tag, m.z_dim))
    return m, enc, dec, x, y, eps, gu.load(tag + ".npz")


def build_imspec(tag):
    """(net [atomai_b200 SignalED, CPU], sd, x, target, golden)."""
    from atomai_b200.nets import init_imspec_model
    c = cases.IMSPEC_CASES[tag]
    net, _ = init_imspec_model(c["in_dim"], c["out_dim"], 4, **c["kw"])
    sd = _seed(net, c["seed"])
    x, y = (torch.from_numpy(a) for a in cases.imspec_inputs(tag))
    return net, sd, x, y, gu.load(tag + ".npz")


def check_grads(named_grads, gold):
    for key, g in named_grads:
        ref = gold[f"grad/{key}"]
        got = gu.sample_flat(g, 97) if g.size > 4096 else g
        gn = float(gold[f"gradnorm/{key}"])
        assert np.abs(got.reshape(-1) - ref.reshape(-1)).max() <= 2e-3 * gn / np.sqrt(g.size) * 30 + 1e-6, key


@pytest.mark.parametrize("tag", list(cases.CVAE_CASES))
def test_cvae_oracle_matches_reference(tag):
    c = cases.CVAE_CASES[tag]
    m, enc, dec, x, y, eps, gold = build_cvae(tag)
    enc = {k: v.clone().requires_grad_(True) for k, v in enc.items()}
    dec = {k: v.clone().requires_grad_(True) for k, v in dec.items()}
    oh = ref.onehot(y, cases.NB_CLASSES)
    conv = bool(c["kw"].get("conv_encoder"))
    if c["kind"] == "rvae":
        elbo, zm, zl, xr = ref.crvae_forward(
            x, eps, oh, enc, dec, cases.HW, conv,
            translation=c["kw"].get("translation", True), skip=c["kw"].get("skip", False))
    else:
        elbo, zm, zl, xr = ref.cvae_forward(x, eps, oh, enc, dec, cases.HW, conv)
    np.testing.assert_allclose(zm.detach().numpy(), gold["z_mean"], atol=2e-5)
    np.testing.assert_allclose(zl.detach().numpy(), gold["z_logsd"], atol=2e-5)
    np.testing.assert_allclose(xr.detach().numpy(), gold["x_reconstr"], atol=5e-5)
    assert abs(elbo.item() - float(gold["elbo"])) < 1e-4 * abs(float(gold["elbo"]))
    (-elbo).backward()
    check_grads([(f"{p}.{k}", v.grad.numpy()) for p, sd in (("encoder", enc), ("decoder", dec))
                 for k, v in sd.items()], gold)


@pytest.mark.parametrize("tag", list(cases.IMSPEC_CASES))
def test_imspec_options_oracle_matches_reference(tag):
    c = cases.IMSPEC_CASES[tag]
    net, sd, x, y, gold = build_imspec(tag)
    kw = dict(nbf=c["kw"]["nbfilters_decoder"], downsampling=c["kw"].get("encoder_downsampling", 0),
              upsampling=c["kw"].get("decoder_upsampling", False))
    out = c["out_dim"]
    with torch.no_grad():
        pe = ref.signal_ed(x, sd, out, **kw)
    np.testing.assert_allclose(pe.numpy(), gold["pred_eval"], atol=5e-5)
    leaves = {k: (v.clone().requires_grad_(True) if v.dtype.is_floating_point and "running" not in k
                  else v.clone()) for k, v in sd.items()}
    pt = ref.signal_ed(x, leaves, out, training=True, new_stats={}, **kw)
    np.testing.assert_allclose(pt.detach().numpy(), gold["pred_train"], atol=1e-4)
    loss = torch.nn.functional.mse_loss(pt, y)
    assert abs(loss.item() - float(gold["loss_train"])) < 1e-5
    loss.backward()
    check_grads([(f"net.{k}", v.grad.numpy()) for k, v in leaves.items() if v.requires_grad], gold)
