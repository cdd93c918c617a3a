"""
Cases of the DenoisingAutoencoder goldens, shared by make_golden_dae.py (which runs the unmodified
reference) and the parity tests.  Inputs are seeded: clean = golden_utils.images, noisy = clean +
N(0, 0.1^2) noise; the loss is the MSE between the network output for `noisy` and `clean`.
"""
import numpy as np

import golden_utils as gu

DAE_CASES = {
    # default config: 1->8 and 16->8 full-resolution layers on the thin-channel kernels
    "default_64": dict(kw={}, n=4, h=64, w=64, seed=900),
    "bn_bilinear_64": dict(kw=dict(use_batch_norm=True, upsampling_mode="bilinear"),
                           n=4, h=64, w=64, seed=910),
    # >= 16 channels everywhere: every 3x3 convolution, full resolution included, on wgmma
    "wide_128": dict(kw=dict(encoder_filters=[16, 32, 64, 128],
                             decoder_filters=[128, 64, 32, 16]), n=2, h=64, w=64, seed=920),
    "three_level_32": dict(kw=dict(encoder_filters=[8, 16, 32], decoder_filters=[32, 16, 8],
                                   encoder_layers=[1, 2, 2], decoder_layers=[2, 2, 1]),
                           n=4, h=32, w=32, seed=930),
}

ADAM_STEPS = 5


def inputs(c):
    """noisy, clean: float32 (n, 1, h, w)."""
    clean = gu.images(c["seed"] + 1, c["n"], c["h"], c["w"])[:, None]
    noise = np.random.RandomState(c["seed"] + 2).normal(0, 0.1, clean.shape).astype(np.float32)
    return clean + noise, clean


def sampled(a):
    """What the goldens store of a parameter-sized array (strided sample above 4096 entries)."""
    return gu.sample_flat(a, 97) if a.size > 4096 else a


# tiny reference-written checkpoint (dae_fit.tar): reference DenoisingAutoencoder.fit with swa (the
# reference averages the last 30 cycles and needs at least that many)
CKPT = dict(kw=dict(encoder_filters=[8, 16, 16], decoder_filters=[16, 16, 8],
                    encoder_layers=[1, 1, 1], decoder_layers=[1, 1, 1]),
            n=24, h=32, w=32, cycles=30, batch_size=8, seed=950)
