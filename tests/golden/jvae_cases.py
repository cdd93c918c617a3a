"""
Cases of the jVAE / jrVAE goldens, shared by make_golden_jvae.py (which runs the unmodified
reference) and the parity tests.  num_iter is the count before the step (the step adds one); the
capacities are the reference's defaults [5.0, 25000, 30], so the continuous cap is 5 * (num_iter + 1)
/ 25000 and the discrete cap is clipped by sum(log D) in jvae_conv_32 and jrvae_fc_32.
"""
import numpy as np

import golden_utils as gu

HW = (32, 32)
N = 8

JVAE_CASES = {
    "jvae_fc_32": dict(kind="jvae", conv=False, discrete=[4], tau=0.67, num_iter=3000, seed=800),
    "jvae_conv_32": dict(kind="jvae", conv=True, discrete=[3, 5], tau=0.5, num_iter=20000,
                         seed=810),
    "jrvae_conv_32": dict(kind="jrvae", conv=True, discrete=[4], tau=0.67, num_iter=6000,
                          translation=True, phi_prior=0.1, dx_prior=0.15, seed=820),
    "jrvae_fc_32": dict(kind="jrvae", conv=False, discrete=[3, 2], tau=0.67, num_iter=15000,
                        translation=False, skip=True, phi_prior=0.2, seed=830),
}


def model_kwargs(c):
    """Constructor kwargs of a case (the same for the reference and atomai_b200)."""
    kw = dict(latent_dim=2, discrete_dim=list(c["discrete"]), conv_encoder=c["conv"])
    if c["kind"] == "jvae":
        kw["conv_decoder"] = c["conv"]
    else:
        kw["translation"] = c["translation"]
        kw["skip"] = c.get("skip", False)
    return kw


def inputs(c, zdim_cont):
    """x (N, H, W), eps (N, latent + coord), u (N, sum D), all float32."""
    x = gu.images(c["seed"] + 2, N, *HW)
    eps = np.random.RandomState(c["seed"] + 3).randn(N, zdim_cont).astype(np.float32)
    u = np.random.RandomState(c["seed"] + 4).rand(N, sum(c["discrete"])).astype(np.float32)
    return x, eps, u


# tiny reference-written jrVAE checkpoint (jrvae_12.tar): 12 x 12 input, 8 hidden units, one cycle
CKPT = dict(in_dim=(12, 12), latent_dim=2, discrete_dim=[3], numhidden_encoder=8,
            numhidden_decoder=8, n=32, batch_size=8, seed=850)
