"""
TEST INFRASTRUCTURE — CPU restatement (plain torch fp32 functional ops) of the reference's
class-conditioned VAE / rVAE and of ImSpec's encoder_downsampling / decoder_upsampling, built on
the pieces of oracle/vae_ref.py.  Only tests/ may import it.  Parity status: PINNED by
tests/test_oracle_ed_options.py against goldens produced by the unmodified reference
(tests/golden/make_golden_ed_options.py).
"""
from typing import Optional

import torch
import torch.nn.functional as F

from .nets_ref import _conv, conv_block, dilated_block
from .vae_ref import (SD, conv_decoder, conv_encoder, fc_decoder, fc_encoder, imcoordgrid,
                      rvae_elbo, vae_elbo)


def onehot(y, nb_classes: int):
    """to_onehot — atomai/utils/preproc.py:916-930: (B,) labels -> (B, nb_classes) float."""
    return torch.zeros(len(y), nb_classes).scatter_(1, y.view(-1, 1), 1.0)


def r_decoder(z, phi, dx, sd: SD, hw, num_layers=2, skip=False):
    """transform_coordinates + rDecoderNet.forward — atomai/utils/coords.py:57-83,
    atomai/nets/ed.py:626-642, 672-687 (c=1).  skip=True: no tanh after coord_latent, and its
    output is added after every (Linear, Tanh) pair."""
    b = z.shape[0]
    grid = imcoordgrid(hw).expand(b, -1, -1)
    c, s = torch.cos(phi), torch.sin(phi)
    rot = torch.stack([torch.stack([c, s], 1), torch.stack([-s, c], 1)], 1)
    coord = torch.bmm(grid, rot)
    if dx is not None:
        coord = coord + dx.unsqueeze(1)
    h = F.linear(coord.reshape(-1, 2), sd["coord_latent.fc_coord.weight"],
                 sd["coord_latent.fc_coord.bias"]).reshape(b, hw[0] * hw[1], -1)
    h = h + F.linear(z, sd["coord_latent.fc_latent.weight"]).unsqueeze(1)
    if not skip:
        h = torch.tanh(h)
    h = h.reshape(b * hw[0] * hw[1], -1)
    res = h
    for i in range(num_layers):
        h = torch.tanh(F.linear(h, sd[f"fc_decoder.{2*i}.weight"], sd[f"fc_decoder.{2*i}.bias"]))
        if skip:
            h = h + res
    return F.linear(h, sd["out.weight"], sd["out.bias"]).reshape(b, *hw)


def cvae_forward(x, eps, y_onehot, enc: SD, dec: SD, hw, conv: bool, hidden=128):
    """Class-conditioned VAE.forward_compute_elbo — atomai/models/dgm/vae.py:661-687 with injected
    noise: the one-hot label is appended to the decoder input."""
    z_mean, z_logsd = (conv_encoder if conv else fc_encoder)(x, enc)
    z = torch.cat((z_mean + torch.exp(z_logsd) * eps, y_onehot), -1)
    x_rec = conv_decoder(z, dec, hw, hidden) if conv else fc_decoder(z, dec, hw)
    return vae_elbo(x, x_rec, z_mean, z_logsd), z_mean, z_logsd, x_rec


def crvae_forward(x, eps, y_onehot, enc: SD, dec: SD, hw, conv_enc: bool, translation=True,
                  skip=False, dx_prior=0.1):
    """Class-conditioned rVAE.forward_compute_elbo — atomai/models/dgm/rvae.py:110-147 with
    injected noise: the one-hot label is appended to the content latents."""
    z_mean, z_logsd = (conv_encoder if conv_enc else fc_encoder)(x, enc)
    z = z_mean + torch.exp(z_logsd) * eps
    zc, dx = (z[:, 3:], z[:, 1:3] * dx_prior) if translation else (z[:, 1:], None)
    x_rec = r_decoder(torch.cat((zc, y_onehot), -1), z[:, 0], dx, dec, hw, skip=skip)
    return rvae_elbo(x, x_rec, z_mean, z_logsd), z_mean, z_logsd, x_rec


def signal_ed(x, sd: SD, out_dims, nb_enc=3, nb_dec=4, nbf=64, training=False,
              new_stats: Optional[dict] = None, downsampling: int = 0, upsampling: bool = False):
    """SignalED.forward with the resampling options — atomai/nets/ed.py:66-79, 144-157, 223-228.
    `out_dims`: (length,) of a spectrum target or (h, w) of an image target.  downsampling = s:
    average pool (s, floor) of the input before the encoder; upsampling: fc to dims // 4, then
    (ConvBlock, nearest x2) twice."""
    kw = dict(training=training, new_stats=new_stats)
    dims = tuple(out_dims)
    if downsampling:
        pool = F.avg_pool1d if x.ndim == 3 else F.avg_pool2d
        x = pool(x, downsampling, downsampling)
    h = conv_block(x, sd, "encoder.conv", nb_enc, True, 0.1, **kw)
    z = F.linear(h.reshape(h.shape[0], -1), sd["encoder.fc.weight"], sd["encoder.fc.bias"])
    if upsampling:
        dims = tuple(d // 4 for d in dims)
    h = F.linear(z, sd["decoder.fc.weight"], sd["decoder.fc.bias"]).reshape(-1, nbf, *dims)
    if upsampling:
        for name in ("decoder.deconv1", "decoder.deconv2"):
            h = conv_block(h, sd, name, 1, True, 0.1, **kw)
            h = F.interpolate(h, scale_factor=2, mode="nearest")
    h = dilated_block(h, sd, "decoder.dilblock", list(range(1, nb_dec + 1)), True, 0.1, **kw)
    h = conv_block(h, sd, "decoder.conv", 1, True, 0.1, **kw)
    return _conv(h, sd, "decoder.out")
