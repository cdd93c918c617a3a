"""jVAE / jrVAE without a GPU: the oracle (oracle/jvae_ref.py) against goldens produced by the
unmodified reference (tests/golden/make_golden_jvae.py), module tree and state_dict keys, z_dim and
metadict, loading a reference-written checkpoint, the C ABI's argument checks and the resource
usage of the joint-latent kernels."""
import ctypes
import os
import re
import shutil
import subprocess
from collections import OrderedDict

import numpy as np
import pytest
import torch

import golden_utils as gu
from jvae_cases import CKPT, HW, JVAE_CASES, inputs, model_kwargs
from oracle import jvae_ref

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def build_jvae(name):
    """(model [atomai_b200, on the default device], enc sd, dec sd, x, eps, u, golden)."""
    from atomai_b200.models import jrVAE, jVAE
    c = JVAE_CASES[name]
    m = (jVAE if c["kind"] == "jvae" else jrVAE)(HW, **model_kwargs(c))
    sds = []
    for net, seed in ((m.encoder_net, c["seed"]), (m.decoder_net, c["seed"] + 1)):
        shapes = OrderedDict((k, tuple(v.shape)) for k, v in net.state_dict().items())
        sd = OrderedDict((k, torch.from_numpy(v)) for k, v in gu.fill_state_dict(shapes, seed).items())
        net.load_state_dict(sd)
        sds.append(sd)
    x, eps, u = (torch.from_numpy(a) for a in inputs(c, m.z_dim - sum(c["discrete"])))
    m.kdict_["temperature"] = c["tau"]
    m.kdict_["num_iter"] = c["num_iter"]
    if c["kind"] == "jrvae":
        m.dx_prior = c.get("dx_prior", 0.1)
        m.kdict_["phi_prior"] = c["phi_prior"]
    return m, sds[0], sds[1], x, eps, u, gu.load(name + ".npz")


@pytest.mark.parametrize("name", list(JVAE_CASES))
def test_jvae_oracle_matches_reference(name):
    c = JVAE_CASES[name]
    m, enc, dec, x, eps, u, gold = build_jvae(name)
    enc = {k: v.clone().requires_grad_(True) for k, v in enc.items()}
    dec = {k: v.clone().requires_grad_(True) for k, v in dec.items()}
    elbo, zm, zl, alpha, zd, xr = jvae_ref.joint_forward(x, eps, u, enc, dec, HW, c)
    np.testing.assert_allclose(zm.detach().numpy(), gold["z_mean"], atol=2e-5)
    np.testing.assert_allclose(zl.detach().numpy(), gold["z_logsd"], atol=2e-5)
    np.testing.assert_allclose(alpha.detach().numpy(), gold["alphas"], atol=1e-6)
    np.testing.assert_allclose(zd.detach().numpy(), gold["z_disc"], atol=1e-5)
    np.testing.assert_allclose(xr.detach().numpy(), gold["x_reconstr"], atol=5e-5)
    assert abs(elbo.item() - float(gold["elbo"])) < 1e-5 * abs(float(gold["elbo"]))
    (-elbo).backward()
    for pref, sd in (("encoder", enc), ("decoder", dec)):
        for k, p in sd.items():
            g = p.grad.numpy()
            ref = gold[f"grad/{pref}.{k}"]
            got = gu.sample_flat(g, 97) if g.size > 4096 else g
            gn = float(gold[f"gradnorm/{pref}.{k}"])
            assert np.abs(got.reshape(-1) - ref.reshape(-1)).max() <= 2e-3 * gn / np.sqrt(g.size) * 30 + 1e-6, k


@pytest.mark.parametrize("name", list(JVAE_CASES))
def test_module_tree_and_state_dict_keys_match_reference(name):
    from atomai_b200.nets import jconvEncoderNet, jfcEncoderNet
    c = JVAE_CASES[name]
    m, *_, gold = build_jvae(name)
    enc = m.encoder_net
    assert isinstance(enc, jconvEncoderNet if c["conv"] else jfcEncoderNet)
    trunk = "conv" if c["conv"] else "dense"
    assert [n for n, _ in enc.named_children()][:4] == [trunk, "fc11", "fc12", "fc13"]
    assert [h.out_features for h in enc.fc13] == c["discrete"]
    for pref, net in (("encoder", m.encoder_net), ("decoder", m.decoder_net)):
        keys = [k for k, _ in net.named_parameters()]
        ref = [k[len("grad/") + len(pref) + 1:] for k in gold.files if k.startswith(f"grad/{pref}.")]
        assert keys == ref, (pref, keys, ref)
        for k, p in net.named_parameters():
            if p.numel() <= 4096:
                assert tuple(p.shape) == gold[f"grad/{pref}.{k}"].shape, k


def test_z_dim_and_metadict():
    from atomai_b200.models import jrVAE, jVAE
    m = jVAE((16, 16), latent_dim=3, discrete_dim=[4, 2], nb_classes=5)
    assert m.z_dim == 3 + 6 and m.coord == 0 and m.discrete_dim == [4, 2]
    assert m.metadict["discrete_dim"] == [4, 2] and m.metadict["nb_classes"] == 5
    assert m.decoder_net.decoder[0].in_features == 3 + 6          # nb_classes is dropped
    assert m.encoder_net.fc11.out_features == 3
    r = jrVAE((16, 16), latent_dim=2, discrete_dim=[5], translation=False)
    assert r.z_dim == 2 + 1 + 5 and r.coord == 1
    assert r.encoder_net.fc11.out_features == 3
    assert r.decoder_net.coord_latent.fc_latent.in_features == 2 + 5
    assert r.kdict_["num_iter"] == 0 and r.metadict["coord"] == 1
    assert jrVAE((16, 16)).z_dim == 2 + 3 + 2                   # reference default discrete_dim=[2]


def test_load_reference_checkpoint():
    from atomai_b200.models import jrVAE, load_model
    path = os.path.join(gu.GOLDEN_DIR, "jrvae_12.tar")
    ck = torch.load(path, map_location="cpu", weights_only=False)
    m = load_model(path)
    assert type(m) is jrVAE and m.translation and m.coord == 3
    assert m.discrete_dim == CKPT["discrete_dim"] and tuple(m.in_dim) == CKPT["in_dim"]
    assert m.kdict_["num_iter"] == ck["num_iter"] == int(gu.load("jrvae_12_encode.npz")["num_iter"])
    for net, key in ((m.encoder_net, "encoder"), (m.decoder_net, "decoder")):
        sd = net.state_dict()
        assert list(sd) == list(ck[key])
        for k, v in ck[key].items():
            assert torch.equal(sd[k].cpu(), v.cpu()), k


def test_joint_capacity_matches_reference_rule():
    from atomai_b200.losses_metrics import kld_discrete
    from atomai_b200.losses_metrics.vi_losses import _joint_infocapacity
    a = torch.softmax(torch.randn(7, 5, dtype=torch.float64), 1)
    assert torch.allclose(kld_discrete(a), jvae_ref.kld_discrete(a).view(1))
    kc, kd = torch.tensor(1.5, dtype=torch.float64), torch.tensor(2.0, dtype=torch.float64)
    for num_iter in (0, 100, 20000, 10 ** 6):
        got = _joint_infocapacity(kc, [5.0, 25000, 30], kd, [5.0, 25000, 30], [3, 5], num_iter)
        ref = jvae_ref.capacity_terms(kc, kd, [3, 5], num_iter)
        assert all(torch.allclose(g, r) for g, r in zip(got, ref))
    # the discrete cap is clipped by sum(log D): at 10**6 iterations 30 * |log 3 + log 5 - 2|
    _, d = _joint_infocapacity(kc, [5.0, 25000, 30], kd, [5.0, 25000, 30], [3, 5], 10 ** 6)
    assert abs(float(d) - 30 * abs(np.log(15) - 2.0)) < 1e-12
    # |x| has gradient 0 at 0, as torch.abs
    k0 = torch.tensor(0.0, requires_grad=True)
    c, _ = _joint_infocapacity(k0, [5.0, 25000, 30], kd, [5.0, 25000, 30], [2], 0)
    c.backward()
    assert float(k0.grad) == 0.0


def test_exports():
    import atomai_b200.losses_metrics as lm
    import atomai_b200.models as models
    import atomai_b200.models.dgm as dgm
    import atomai_b200.nets as nets
    from atomai_b200 import _C
    for mod, names in ((models, ("jVAE", "jrVAE")), (dgm, ("jVAE", "jrVAE")),
                       (nets, ("jfcEncoderNet", "jconvEncoderNet")),
                       (lm, ("kld_discrete", "joint_vae_loss", "joint_rvae_loss"))):
        for n in names:
            assert n in mod.__all__ and hasattr(mod, n), (mod.__name__, n)
    lib = _C.lib()
    for s in ("atomai_b200_jlatent_fwd", "atomai_b200_jlatent_bwd"):
        assert hasattr(lib, s) and s in _C.SIGNATURES
    assert ctypes.sizeof(_C.JLat) == (4 + 64) * 4 + 3 * 4


def _status(desc, mode=1):
    from atomai_b200 import _C
    lib = _C.lib()
    p = 16   # any non-null address: the checks fail before anything is dereferenced or launched
    return lib.atomai_b200_jlatent_fwd(ctypes.byref(desc), mode, p, p, p, p, None, 0, p, p, p, p,
                                       None, None), lib.atomai_b200_last_error()


def test_out_of_limit_arguments_return_status_without_gpu():
    from atomai_b200 import ops
    good = dict(B=4, Dc=5, coord=3, heads=[4], tau=0.67)
    bad = [dict(heads=[40, 25]), dict(heads=[3, 0]), dict(Dc=33, coord=0), dict(coord=2),
           dict(Dc=3, coord=3), dict(tau=0.0), dict(tau=-1.0), dict(B=-1)]
    for b in bad:
        kw = dict(good, **b)
        d = ops.jlat_desc(kw["B"], kw["Dc"], kw["coord"], kw["heads"], kw["tau"])
        rc, msg = _status(d)
        assert rc != 0 and b"jlatent" in msg, (b, msg)
        with pytest.raises(ValueError):
            ops._check_args(rc)
    assert _status(ops.jlat_desc(4, 5, 3, [4], 0.67), mode=7)[0] != 0
    with pytest.raises(ValueError):
        ops.jlat_desc(4, 5, 3, [1] * 65, 0.67)
    # B = 0 at the limits (Dc = 32, sum D = 64) is accepted and launches nothing
    assert _status(ops.jlat_desc(0, 32, 3, [32, 32], 0.67))[0] == 0


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_joint_latent_kernels_have_no_stack():
    from atomai_b200 import _C
    res = subprocess.run([CUOBJDUMP, "-res-usage", _C.build()], capture_output=True, text=True).stdout
    found, name = {}, None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name and "jlatent" in name:
            found[name] = int(m.group(2))
            name = None
    assert len(found) == 2, found
    assert all(v == 0 for v in found.values()), found
