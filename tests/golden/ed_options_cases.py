"""Cases of make_golden_ed_options.py and their seeded inputs (shared with the tests): the
class-conditioned VAE / rVAE and ImSpec with encoder_downsampling / 1-D decoder_upsampling."""
import numpy as np

import golden_utils as gu

HW = (32, 32)
N = 8
NB_CLASSES = 3

CVAE_CASES = {
    "cvae_fc_32": dict(kind="vae", seed=800, kw={}),
    "cvae_conv_32": dict(kind="vae", seed=810, kw=dict(conv_encoder=True, conv_decoder=True)),
    "crvae_conv_32": dict(kind="rvae", seed=820, kw=dict(conv_encoder=True)),
    "crvae_notrans_32": dict(kind="rvae", seed=830, kw=dict(translation=False)),
    "crvae_skip_32": dict(kind="rvae", seed=840, kw=dict(skip=True)),
}

IMSPEC_CASES = {
    # image side 15: the 2x2 average pool drops the last row and column
    "im2spec_ds2_up_15_32": dict(in_dim=(15, 15), out_dim=(32,), seed=850, n=6,
                                 kw=dict(encoder_downsampling=2, decoder_upsampling=True,
                                         nbfilters_decoder=8)),
    # spectrum length 50: the window-3 average pool drops the last two points
    "spec2im_ds3_50_8": dict(in_dim=(50,), out_dim=(8, 8), seed=860, n=6,
                             kw=dict(encoder_downsampling=3, nbfilters_decoder=8)),
}

CKPT = dict(in_dim=(16, 16), seed=870, kw=dict(numhidden_encoder=32, numhidden_decoder=32))


def cvae_inputs(tag, z_dim):
    """(x (N, 32, 32), labels (N,) int64 with every class present, eps (N, z_dim))."""
    s = CVAE_CASES[tag]["seed"]
    x = gu.images(s + 2, N, *HW)
    y = np.random.RandomState(s + 4).randint(0, NB_CLASSES, N).astype(np.int64)
    y[:NB_CLASSES] = np.arange(NB_CLASSES)
    eps = np.random.RandomState(s + 3).randn(N, z_dim).astype(np.float32)
    return x, y, eps


def imspec_inputs(tag):
    """(x (n, 1, *in_dim), target (n, 1, *out_dim)) in the reference's channel-first layout."""
    c = IMSPEC_CASES[tag]
    s, n = c["seed"], c["n"]
    if len(c["in_dim"]) == 2:
        x = gu.images(s + 1, n, *c["in_dim"])[:, None]
    else:
        x = np.random.RandomState(s + 1).rand(n, 1, *c["in_dim"]).astype(np.float32)
    y = np.random.RandomState(s + 2).rand(n, 1, *c["out_dim"]).astype(np.float32)
    return x, y


def ckpt_inputs():
    """(z (5, 2), labels (5,)) decoded from the checkpoint."""
    rs = np.random.RandomState(CKPT["seed"] + 2)
    return rs.randn(5, 2).astype(np.float32), np.array([0, 1, 2, 1, 0], np.int64)
