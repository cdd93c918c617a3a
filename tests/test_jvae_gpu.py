"""jVAE / jrVAE on the GPU: parity with the reference's goldens (tests/golden/make_golden_jvae.py)
in fp32 and tf32 math with the tolerances of test_vae_gpu.py, the fused joint-latent kernels
against a float64 restatement of the reference's expressions (oracle/jvae_ref.py), their limits,
determinism and Gumbel-max sampling, and the model API (fit / encode / decode / reconstruct /
save / load)."""
import os

import numpy as np
import pytest
import torch

import golden_utils as gu
from jvae_cases import HW, JVAE_CASES
from oracle import jvae_ref
from test_jvae import build_jvae
from test_vae_gpu import grad_rel, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", list(JVAE_CASES))
def test_jvae_forward_backward(cuda, name, math):
    import atomai_b200 as ab
    from atomai_b200.losses_metrics.vi_losses import joint_latent
    ab.set_math(math)
    c = JVAE_CASES[name]
    m, enc, dec, x, eps, u, gold = build_jvae(name)
    assert m.device == "cuda"
    x, eps, u = x.to(cuda), eps.to(cuda), u.to(cuda)
    tol = 1e-4 if math == "fp32" else 2e-3
    m.encoder_net.train(); m.decoder_net.train()
    elbo = m.forward_compute_elbo(x, eps=eps, u=u)
    (-elbo).backward()
    assert m.kdict_["num_iter"] == c["num_iter"] + 1
    assert abs(elbo.item() - float(gold["elbo"])) <= tol * abs(float(gold["elbo"]))
    with torch.no_grad():
        zm, zl, *alphas = m.encoder_net(x)
        _, _, logits = m.encoder_net.heads(x)
        _, zdec, phi, dx, _ = joint_latent(zm, zl, logits, c["discrete"], c["tau"], eps, u,
                                           coord=m.coord, phi_prior=c.get("phi_prior", 0.1),
                                           dx_prior=c.get("dx_prior", 0.1))
        if m.coord:
            xr = m.decoder_net.decode(zdec, phi, dx if m.coord == 3 else None)
        else:
            xr = m.decoder_net(zdec)
    assert [a.shape[1] for a in alphas] == c["discrete"]
    assert rel(zm.cpu().numpy(), gold["z_mean"]) <= tol
    assert rel(zl.cpu().numpy(), gold["z_logsd"]) <= tol
    assert rel(torch.cat(alphas, 1).cpu().numpy(), gold["alphas"]) <= tol
    assert rel(zdec[:, -sum(c["discrete"]):].cpu().numpy(), gold["z_disc"]) <= tol * 3
    assert xr.shape == (x.shape[0], *HW)
    assert rel(xr.cpu().numpy(), gold["x_reconstr"]) <= tol * 3
    g = grad_rel([("encoder", m.encoder_net), ("decoder", m.decoder_net)], gold)
    assert g <= (2e-3 if math == "fp32" else 5e-2), g


def _rel(a, ref):
    a, ref = a.detach().double(), ref.detach().double()
    return float((a - ref).abs().max() / max(float(ref.abs().max()), 1e-6))


HEADS = [[1], [2], [10], [3, 5, 7], [30, 34]]        # the last one at the sum(D) <= 64 limit


@pytest.mark.parametrize("B", [1, 7, 100, 1000])
@pytest.mark.parametrize("hi", range(len(HEADS)))
def test_fused_kernels_match_float64(cuda, B, hi):
    """Forward outputs and all input gradients of the fused block against the reference's
    expressions evaluated in float64, for jVAE (coord 0) and jrVAE (coord 1 and 3) layouts."""
    from atomai_b200.losses_metrics.vi_losses import joint_latent
    heads = HEADS[hi]
    D = sum(heads)
    gen = torch.Generator(device="cpu").manual_seed(1000 * B + hi)
    for ti, tau in enumerate((0.1, 0.67, 2.0)):
        coord = (0, 1, 3)[(hi + ti) % 3]
        Dc = 32 if hi == len(HEADS) - 1 else 2 + coord
        r = lambda *s: torch.randn(*s, generator=gen)                                # noqa: E731
        mu, ls, logits = r(B, Dc), 0.5 * r(B, Dc), 3.0 * r(B, D)
        eps, u = r(B, Dc), torch.rand(B, D, generator=gen)
        ins = [t.to(cuda).requires_grad_(True) for t in (mu, ls, logits)]
        outs = joint_latent(ins[0], ins[1], ins[2], heads, tau, eps.to(cuda), u.to(cuda),
                            coord=coord, phi_prior=0.3, dx_prior=0.2)
        ref_in = [t.double().to(cuda).requires_grad_(True) for t in (mu, ls, logits)]
        a, zdec, phi, dx, kc, kd = jvae_ref.joint_latent(
            ref_in[0], ref_in[1], ref_in[2], heads, tau, eps.double().to(cuda),
            u.double().to(cuda), coord, 0.3, 0.2)
        refs = [a, zdec, phi, dx, torch.stack([kc, kd])]
        got = [outs[0], outs[1], outs[2] if coord else None, outs[3] if coord == 3 else None, outs[4]]
        loss, ref_loss = 0.0, 0.0
        for k, (g, rf) in enumerate(zip(got, refs)):
            if rf is None:
                continue
            assert g.shape == rf.shape, (k, g.shape, rf.shape)
            assert _rel(g, rf) <= 1e-5, (k, tau, coord, _rel(g, rf))
            w = torch.randn(rf.shape, generator=gen).to(cuda)
            loss = loss + (g * w).sum()
            ref_loss = ref_loss + (rf * w.double()).sum()
        loss.backward()
        ref_loss.backward()
        for k, (g, rf) in enumerate(zip(ins, ref_in)):
            assert _rel(g.grad, rf.grad) <= 1e-5, (k, tau, coord, _rel(g.grad, rf.grad))


def test_over_limit_input_raises(cuda):
    from atomai_b200.losses_metrics.vi_losses import joint_alphas, joint_latent
    B = 4
    ok = dict(mu=torch.zeros(B, 5, device=cuda), logsd=torch.zeros(B, 5, device=cuda))
    with pytest.raises(ValueError):
        joint_latent(ok["mu"], ok["logsd"], torch.zeros(B, 65, device=cuda), [65], 0.5,
                     torch.zeros(B, 5, device=cuda))
    with pytest.raises(ValueError):
        joint_latent(torch.zeros(B, 33, device=cuda), torch.zeros(B, 33, device=cuda),
                     torch.zeros(B, 4, device=cuda), [4], 0.5, torch.zeros(B, 33, device=cuda))
    with pytest.raises(ValueError):
        joint_latent(ok["mu"], ok["logsd"], torch.zeros(B, 4, device=cuda), [4], 0.0,
                     torch.zeros(B, 5, device=cuda))
    with pytest.raises(ValueError):
        joint_latent(ok["mu"], ok["logsd"], torch.zeros(B, 4, device=cuda), [3], 0.5,
                     torch.zeros(B, 5, device=cuda))
    with pytest.raises(ValueError):
        joint_alphas(torch.zeros(B, 70, device=cuda), [35, 35])


def test_same_seed_same_bits_other_seed_other_sample(cuda):
    from atomai_b200.losses_metrics.vi_losses import joint_latent
    torch.manual_seed(3)
    B, heads = 1000, [3, 5, 7]
    mu, ls = torch.randn(B, 5, device=cuda), torch.randn(B, 5, device=cuda)
    logits, eps = torch.randn(B, 15, device=cuda), torch.randn(B, 5, device=cuda)
    runs = [joint_latent(mu, ls, logits, heads, 0.67, eps, seed=s, coord=3) for s in (11, 11, 12)]
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    assert not torch.equal(runs[0][1][:, 2:], runs[2][1][:, 2:])
    assert torch.equal(runs[0][4], runs[2][4]) and torch.equal(runs[0][0], runs[2][0])


def test_gumbel_max_property_of_hash_noise(cuda):
    """argmax(log alpha + g) of the hash-generated Gumbel noise is distributed as alpha."""
    from scipy.stats import chisquare
    from atomai_b200.losses_metrics.vi_losses import joint_latent
    alpha = torch.tensor([0.05, 0.1, 0.2, 0.3, 0.35], device=cuda)
    B = 2 ** 16
    logits = torch.log(alpha).expand(B, -1).contiguous()
    z = torch.zeros(B, 1, device=cuda)
    _, zdec, *_ = joint_latent(z, z, logits, [5], 1.0, z, seed=2024)
    counts = torch.bincount(zdec[:, 1:].argmax(1), minlength=5).cpu().numpy()
    p = chisquare(counts, (alpha.cpu().numpy() * B)).pvalue
    assert p > 1e-3, (counts, p)


def _api_checks(m, X):
    zm, zs, alphas = m.encode(X[:10])
    zc = m.z_dim - sum(m.discrete_dim)
    assert zm.shape == (10, zc) and zs.shape == (10, zc) and alphas.shape == (10, sum(m.discrete_dim))
    offs = np.cumsum([0] + m.discrete_dim)
    for h in range(len(m.discrete_dim)):
        np.testing.assert_allclose(alphas[:, offs[h]:offs[h + 1]].sum(1), 1.0, atol=1e-5)
    z = np.concatenate([zm[:, m.coord:], alphas], 1)
    assert m.decode(z).shape == (10, *m.in_dim)
    assert m.reconstruct(X[:10]).shape == (10, *m.in_dim)
    lab = 0 if len(m.discrete_dim) == 1 else [0] * len(m.discrete_dim)
    assert m.reconstruct(X[:3], label=lab).shape == (3, *m.in_dim)
    with pytest.raises(NotImplementedError):
        m.encode_image_(X[0])


@pytest.mark.parametrize("kind", ["jvae", "jrvae"])
def test_fit_encode_decode_save_load(cuda, tmp_path, kind):
    import atomai_b200 as ab
    from atomai_b200.models import jrVAE, jVAE, load_model
    ab.set_math("tf32")
    X = gu.images(5, 64, 32, 32)
    if kind == "jvae":
        m = jVAE((32, 32), latent_dim=2, discrete_dim=[3, 4], conv_encoder=True,
                 numhidden_encoder=32, numhidden_decoder=32)
    else:
        m = jrVAE((32, 32), latent_dim=2, discrete_dim=[4], conv_encoder=True,
                  numhidden_encoder=32, numhidden_decoder=32)
    f = str(tmp_path / kind)
    m.fit(X, training_cycles=3, batch_size=16, filename=f)
    hist = m.loss_history["train_loss"]
    assert len(hist) == 3 and hist[-1] > hist[0]          # ELBO increases
    assert m.kdict_["num_iter"] == 12 and m.metadict["num_iter"] == 12
    _api_checks(m, X)
    m2 = load_model(f + ".tar")
    assert type(m2) is type(m) and m2.kdict_["num_iter"] == 12
    for a, b in zip(m.encode(X[:10]), m2.encode(X[:10])):
        # (the skinny head GEMM adds its k-slices with atomics: last-bit run-to-run differences)
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)


def test_ce_loss_trains_and_sets_sigmoid_out(cuda, tmp_path):
    from atomai_b200.models import jVAE
    X = (gu.images(3, 64, 16, 16) > 0.5).astype(np.float32)
    m = jVAE((16, 16), latent_dim=2, discrete_dim=[3], seed=1)
    m.fit(X, training_cycles=2, batch_size=16, loss="ce", temperature=0.5,
          filename=str(tmp_path / "jce"))
    assert m.sigmoid_out and m.metadict["sigmoid_out"] and m.kdict_["temperature"] == 0.5
    assert np.isfinite(m.loss_history["train_loss"]).all()
    out = m.decode(np.zeros((2, 5), np.float32))
    assert out.min() >= 0 and out.max() <= 1


def test_reference_checkpoint_encodes_like_the_reference(cuda):
    from atomai_b200.models import load_model
    ref = gu.load("jrvae_12_encode.npz")
    m = load_model(os.path.join(gu.GOLDEN_DIR, "jrvae_12.tar"))
    zm, zs, alphas = m.encode(ref["x"], num_batches=1)
    # (the reference's encode returns the log-SD as its second output, this package the SD)
    assert rel(zm, ref["z_mean"]) <= 1e-4 and rel(np.log(zs), ref["z_logsd"]) <= 1e-4
    assert rel(alphas, ref["alphas"]) <= 1e-4
