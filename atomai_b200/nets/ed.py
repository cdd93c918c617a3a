"""
Encoder / decoder networks for ImSpec and the (r)VAEs — constructor signatures, module names and
state_dict layout of the reference (atomai/nets/ed.py:20-228, 231-343, 471-687, 690-790), executed
by the native sm_90a tape (atomai_b200/engine.py).

Each network is one autograd node per call; inside it the ConvBlocks run on the wgmma
convolution kernels, `x.reshape(-1, C*H*W) -> nn.Linear` becomes an NHWC->NCHW transpose kernel +
a split-K GEMM, and the rVAE spatial decoder (coord_latent + transform_coordinates + per-pixel MLP)
is a fused coordinate kernel followed by 1x1 tensor-core convolutions with tanh epilogues.
The joint encoders (jfcEncoderNet / jconvEncoderNet, atomai/nets/ed.py:346-468) add one skinny
Linear per discrete head; their softmax is the joint-latent kernel (losses_metrics/vi_losses.py).
"""
from typing import Dict, List, Optional, Tuple, Type, Union

import numpy as np
import torch
import torch.nn as nn

from .. import engine
from ..engine import ACT_LRELU, ACT_TANH, Act, Tape
from ..losses_metrics.vi_losses import joint_alphas
from .blocks import ConvBlock, DilatedBlock


def _vec(t: torch.Tensor) -> torch.Tensor:
    """(B, K) -> (B,1,1,K) NHWC-shaped view for the tape."""
    return t.reshape(t.shape[0], 1, 1, -1)


def _img_nhwc(x: torch.Tensor, ndim_spatial: int) -> torch.Tensor:
    """Channel-first batch (N,C,H,W) / (N,C,L) -> contiguous NHWC."""
    return engine._to_nhwc(x)


class SignalEncoder(nn.Module):
    """
    Encodes 1D/2D signal into a latent vector (atomai/nets/ed.py:20-79): ConvBlock(nb_layers,
    1 -> nb_filters, lrelu 0.1, BN) -> flatten -> Linear(z_dim).  **batch_norm, **downsampling.
    """
    def __init__(self, signal_dim: Tuple[int], z_dim: int, nb_layers: int, nb_filters: int,
                 **kwargs: int) -> None:
        super(SignalEncoder, self).__init__()
        if isinstance(signal_dim, int):
            signal_dim = (signal_dim,)
        if not 0 < len(signal_dim) < 3:
            raise AssertionError("signal dimensionality must be to 1D or 2D")
        ndim = 2 if len(signal_dim) == 2 else 1
        self.downsample = kwargs.get("downsampling", 0)
        bn = kwargs.get('batch_norm', True)
        if self.downsample:
            signal_dim = [s // self.downsample for s in signal_dim]
        n = int(np.prod(signal_dim))
        self.reshape_ = nb_filters * n
        self.conv = ConvBlock(ndim, nb_layers, 1, nb_filters, lrelu_a=0.1, batch_norm=bn)
        self.fc = nn.Linear(nb_filters * n, z_dim)
        self._ndim = ndim

    def _emit(self, tape: Tape, x: Act) -> Act:
        if self.downsample:         # avg_pool2d(x, s, s) / avg_pool1d on the (N, 1, L, 1) spectrum
            s = self.downsample
            x = tape.avgpool(x, s if self._ndim == 2 else 1, s)
        return tape.linear(tape.flatten(self.conv._emit(tape, x)), self.fc)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = engine.run_multi(self, self._emit, (_img_nhwc(x, 0),))
        return y.reshape(y.shape[0], -1)


class SignalDecoder(nn.Module):
    """
    Decodes a latent vector into 1D/2D signal (atomai/nets/ed.py:82-157): Linear -> reshape
    (nb_filters, *dims) -> [upsampling convs] -> DilatedBlock(dilations 1..nb_layers) ->
    ConvBlock(nb_filters -> 1) -> 1x1 conv.
    """
    def __init__(self, signal_dim: Tuple[int], z_dim: int, nb_layers: int, nb_filters: int,
                 **kwargs: bool) -> None:
        super(SignalDecoder, self).__init__()
        self.upsampling = kwargs.get("upsampling", False)
        bn = kwargs.get('batch_norm', True)
        if isinstance(signal_dim, int):
            signal_dim = (signal_dim,)
        if not 0 < len(signal_dim) < 3:
            raise AssertionError("signal dimensionality must be to 1D or 2D")
        ndim = 2 if len(signal_dim) == 2 else 1
        if self.upsampling:
            signal_dim = [s // 4 for s in signal_dim]
        n = int(np.prod(signal_dim))
        self.reshape_ = (nb_filters, *signal_dim)
        self.fc = nn.Linear(z_dim, nb_filters*n)
        if self.upsampling:
            self.deconv1 = ConvBlock(ndim, 1, nb_filters, nb_filters, lrelu_a=0.1, batch_norm=bn)
            self.deconv2 = ConvBlock(ndim, 1, nb_filters, nb_filters, lrelu_a=0.1, batch_norm=bn)
        self.dilblock = DilatedBlock(
            ndim, nb_filters, nb_filters,
            dilation_values=torch.arange(1, nb_layers + 1).tolist(),
            padding_values=torch.arange(1, nb_layers + 1).tolist(),
            lrelu_a=0.1, batch_norm=bn)
        self.conv = ConvBlock(ndim, 1, nb_filters, 1, lrelu_a=0.1, batch_norm=bn)
        self.out = nn.Conv2d(1, 1, 1) if ndim == 2 else nn.Conv1d(1, 1, 1)
        self._ndim = ndim

    def _emit(self, tape: Tape, z: Act) -> Act:
        c = self.reshape_[0]
        h, w = (self.reshape_[1], self.reshape_[2]) if self._ndim == 2 else (1, self.reshape_[1])
        x = tape.unflatten(tape.linear(z, self.fc), c, h, w)
        if self.upsampling:
            up = (lambda a: tape.upsample(a, "nearest")) if self._ndim == 2 else tape.upsample_w2x
            x = up(self.deconv1._emit(tape, x))
            x = up(self.deconv2._emit(tape, x))
        x = self.dilblock._emit(tape, x)
        x = self.conv._emit(tape, x)
        return tape.conv(x, self.out, None, 1.0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = engine.run_multi(self, self._emit, (_vec(x),))      # (N, H, W, 1)
        y = y.permute(0, 3, 1, 2)
        return y.squeeze(2) if self._ndim == 1 else y


class SignalED(nn.Module):
    """
    Transforms image into spectra (im2spec) and vice versa (spec2im)
    (atomai/nets/ed.py:160-228): SignalEncoder + SignalDecoder, one native graph.
    """
    def __init__(self, feature_dim: Tuple[int], target_dim: Tuple[int], latent_dim: int,
                 nblayers_encoder: int = 3, nblayers_decoder: int = 4,
                 nbfilters_encoder: int = 64, nbfilters_decoder: int = 2,
                 batch_norm: bool = True, encoder_downsampling: int = 0,
                 decoder_upsampling: bool = False) -> None:
        super(SignalED, self).__init__()
        self.encoder = SignalEncoder(feature_dim, latent_dim, nblayers_encoder, nbfilters_encoder,
                                     batch_norm=batch_norm, downsampling=encoder_downsampling)
        self.decoder = SignalDecoder(target_dim, latent_dim, nblayers_decoder, nbfilters_decoder,
                                     batch_norm=batch_norm, upsampling=decoder_upsampling)

    def encode(self, features: torch.Tensor) -> torch.Tensor:
        return self.encoder(features)

    def decode(self, latent: torch.Tensor) -> torch.Tensor:
        return self.decoder(latent)

    def _emit(self, tape: Tape, x: Act) -> Act:
        return self.decoder._emit(tape, self.encoder._emit(tape, x))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = engine.run_multi(self, self._emit, (_img_nhwc(x, 0),))
        y = y.permute(0, 3, 1, 2)
        return y.squeeze(2) if self.decoder._ndim == 1 else y


class convEncoderNet(nn.Module):
    """
    Convolutional encoder/inference network for VAEs (atomai/nets/ed.py:231-289): ConvBlock
    (num_layers, c -> hidden_dim, lrelu 0.1, no BN) -> flatten -> fc11 / fc12.
    Input: (B, H, W) or (B, H, W, C) channel-last, as in the reference.
    """
    def __init__(self, in_dim: Tuple[int], latent_dim: int = 2, num_layers: int = 2,
                 hidden_dim: int = 32, **kwargs: Union[float, bool]) -> None:
        super(convEncoderNet, self).__init__()
        if len(in_dim) not in (1, 2, 3):
            raise ValueError(
                "The input dimensions must be (length,) for 1D data and " +
                "(height, width) or (height, width, channel) for 2D data")
        dim = 2 if len(in_dim) > 1 else 1
        c = in_dim[-1] if len(in_dim) > 2 else 1
        self.conv = ConvBlock(dim, num_layers, c, hidden_dim, lrelu_a=kwargs.get("lrelu_a", 0.1))
        self.reshape_ = int(hidden_dim * np.prod(in_dim[:2]))
        self.fc11 = nn.Linear(self.reshape_, latent_dim)
        self.fc12 = nn.Linear(self.reshape_, latent_dim)
        self._softplus = bool(kwargs.get("softplus_out"))
        self._out = nn.Softplus() if self._softplus else lambda x: x

    def _emit(self, tape: Tape, x: Act):
        flat = tape.flatten(self.conv._emit(tape, x))
        return tape.linear(flat, self.fc11), tape.linear(flat, self.fc12)

    def forward(self, x: torch.Tensor) -> Tuple[torch.Tensor]:
        z_mu, z_ls = engine.run_multi(self, self._emit, (_conv_enc_input(x),))
        z_mu, z_ls = z_mu.reshape(z_mu.shape[0], -1), z_ls.reshape(z_ls.shape[0], -1)
        return z_mu, self._out(z_ls)


def _conv_enc_input(x: torch.Tensor) -> torch.Tensor:
    """Input of the convolutional encoders as a contiguous NHWC batch."""
    if x.ndim == 2:                      # (B, L) spectra -> (B,1,L,1)
        xin = x.reshape(x.shape[0], 1, x.shape[1], 1)
    elif x.ndim == 3:                    # (B, H, W) -> NHWC with C = 1
        xin = x.unsqueeze(-1)
    else:                                # (B, H, W, C) is already channel-last
        xin = x
    return xin.float().contiguous()


class fcEncoderNet(nn.Module):
    """
    MLP encoder/inference network for VAEs (atomai/nets/ed.py:292-343):
    num_layers x (Linear + tanh) -> fc11 / fc12.
    """
    def __init__(self, in_dim: Tuple[int], latent_dim: int = 2, num_layers: int = 2,
                 hidden_dim: int = 32, **kwargs: bool) -> None:
        super(fcEncoderNet, self).__init__()
        dense = []
        for i in range(num_layers):
            input_dim = int(np.prod(in_dim)) if i == 0 else hidden_dim
            dense.extend([nn.Linear(input_dim, hidden_dim), nn.Tanh()])
        self.dense = nn.Sequential(*dense)
        self.reshape_ = hidden_dim
        self.fc11 = nn.Linear(self.reshape_, latent_dim)
        self.fc12 = nn.Linear(self.reshape_, latent_dim)
        self._out = nn.Softplus() if kwargs.get("softplus_out") else lambda x: x

    def _emit(self, tape: Tape, x: Act):
        for m in self.dense:
            if isinstance(m, nn.Linear):
                x = tape.linear(x, m, ACT_TANH)
        return tape.linear(x, self.fc11), tape.linear(x, self.fc12)

    def forward(self, x: torch.Tensor):
        xin = _vec(x.reshape(x.shape[0], -1).float().contiguous())
        z_mu, z_ls = engine.run_multi(self, self._emit, (xin,))
        z_mu, z_ls = z_mu.reshape(z_mu.shape[0], -1), z_ls.reshape(z_ls.shape[0], -1)
        return z_mu, self._out(z_ls)


def _joint_heads(net: nn.Module, xin: torch.Tensor):
    """(z_mean, z_logsd after the optional softplus, the discrete heads' logits concatenated) of a
    joint encoder: trunk, fc11, fc12 and one skinny Linear per head in one native graph."""
    z_mu, z_ls, *logits = engine.run_multi(net, net._emit, (xin,))
    b = z_mu.shape[0]
    return (z_mu.reshape(b, -1), net._out(z_ls.reshape(b, -1)),
            torch.cat([lg.reshape(b, -1) for lg in logits], 1))


class jfcEncoderNet(fcEncoderNet):
    """
    MLP encoder for joint continuous and discrete latents (atomai/nets/ed.py:346-407):
    num_layers x (Linear + tanh) -> fc11 / fc12 / fc13[i] (one Linear per discrete head).
    forward(x) returns [z_mean, z_logsd, alpha_1, ..., alpha_n] as the reference does.
    """
    def __init__(self, in_dim: Tuple[int], latent_dim: int = 2, discrete_dim: List = [1],
                 num_layers: int = 2, hidden_dim: int = 32, **kwargs: bool) -> None:
        super(jfcEncoderNet, self).__init__(in_dim, latent_dim, num_layers, hidden_dim, **kwargs)
        self.fc13 = nn.ModuleList([nn.Linear(self.reshape_, d) for d in discrete_dim])
        self.discrete_dim = [int(d) for d in discrete_dim]

    def _emit(self, tape: Tape, x: Act):
        for m in self.dense:
            if isinstance(m, nn.Linear):
                x = tape.linear(x, m, ACT_TANH)
        return tuple(tape.linear(x, m) for m in (self.fc11, self.fc12, *self.fc13))

    def heads(self, x: torch.Tensor):
        """(z_mean, z_logsd, concatenated head logits): what the joint training step consumes."""
        return _joint_heads(self, _vec(x.reshape(x.shape[0], -1).float().contiguous()))

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        z_mu, z_ls, logits = self.heads(x)
        return [z_mu, z_ls, *torch.split(joint_alphas(logits, self.discrete_dim), self.discrete_dim, 1)]


class jconvEncoderNet(convEncoderNet):
    """
    Convolutional encoder for joint continuous and discrete latents (atomai/nets/ed.py:410-468):
    ConvBlock(num_layers, c -> hidden_dim, lrelu 0.1) -> flatten -> fc11 / fc12 / fc13[i].
    forward(x) returns [z_mean, z_logsd, alpha_1, ..., alpha_n] as the reference does.
    """
    def __init__(self, in_dim: Tuple[int], latent_dim: int = 2, discrete_dim: List = [1],
                 num_layers: int = 2, hidden_dim: int = 32, **kwargs: Union[float, bool]) -> None:
        super(jconvEncoderNet, self).__init__(in_dim, latent_dim, num_layers, hidden_dim, **kwargs)
        self.fc13 = nn.ModuleList([nn.Linear(self.reshape_, d) for d in discrete_dim])
        self.discrete_dim = [int(d) for d in discrete_dim]

    def _emit(self, tape: Tape, x: Act):
        flat = tape.flatten(self.conv._emit(tape, x))
        return tuple(tape.linear(flat, m) for m in (self.fc11, self.fc12, *self.fc13))

    def heads(self, x: torch.Tensor):
        """(z_mean, z_logsd, concatenated head logits): what the joint training step consumes."""
        return _joint_heads(self, _conv_enc_input(x))

    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        z_mu, z_ls, logits = self.heads(x)
        return [z_mu, z_ls, *torch.split(joint_alphas(logits, self.discrete_dim), self.discrete_dim, 1)]


class convDecoderNet(nn.Module):
    """
    Convolutional decoder network for VAEs (atomai/nets/ed.py:471-527): fc_linear (no bias) ->
    reshape (hidden, H, W) -> ConvBlock(lrelu 0.1) -> 1x1 conv -> (B, H, W[, C]).
    """
    def __init__(self, out_dim: Tuple[int], latent_dim: int, num_layers: int = 2,
                 hidden_dim: int = 32, **kwargs: float) -> None:
        super(convDecoderNet, self).__init__()
        if len(out_dim) not in (1, 2, 3):
            raise ValueError(
                "The output dimensions must be (length,) for 1D data and " +
                "(height, width) or (height, width, channel) for 2D data")
        dim = 2 if len(out_dim) > 1 else 1
        c = out_dim[-1] if len(out_dim) > 2 else 1
        self.fc_linear = nn.Linear(latent_dim, int(hidden_dim * np.prod(out_dim[:2])), bias=False)
        self.reshape_ = (hidden_dim, *out_dim[:2])
        self.decoder = ConvBlock(dim, num_layers, hidden_dim, hidden_dim,
                                 lrelu_a=kwargs.get("lrelu_a", 0.1))
        conv_1x1 = nn.Conv2d if dim == 2 else nn.Conv1d
        self.conv_1x1 = conv_1x1(hidden_dim, c, 1, 1, 0)
        self.out_dim = (c, *out_dim[:2])
        self._dim = dim

    def _emit(self, tape: Tape, z: Act) -> Act:
        hid = self.reshape_[0]
        h, w = (self.reshape_[1], self.reshape_[2]) if self._dim == 2 else (1, self.reshape_[1])
        x = tape.unflatten(tape.linear(z, self.fc_linear), hid, h, w)
        x = self.decoder._emit(tape, x)
        return tape.conv(x, self.conv_1x1, None, 1.0)

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        y = engine.run_multi(self, self._emit, (_vec(z.float()),))    # (B, H, W, c)
        if self._dim == 1:
            y = y.squeeze(1)                                          # (B, L, c)
        return y.squeeze(-1) if y.shape[-1] == 1 else y


class fcDecoderNet(nn.Module):
    """
    MLP decoder network for VAEs (atomai/nets/ed.py:530-580):
    num_layers x (Linear + tanh) -> Linear(prod(out_dim)) -> (B, H, W[, C]).
    """
    def __init__(self, out_dim: Tuple[int], latent_dim: int, num_layers: int = 2,
                 hidden_dim: int = 32) -> None:
        super(fcDecoderNet, self).__init__()
        if len(out_dim) not in (1, 2, 3):
            raise ValueError(
                "The output dimensions must be (length,) for 1D data and " +
                "(height, width) or (height, width, channel) for 2D data")
        c = out_dim[-1] if len(out_dim) > 2 else 1
        decoder = []
        for i in range(num_layers):
            hidden_dim_ = latent_dim if i == 0 else hidden_dim
            decoder.extend([nn.Linear(hidden_dim_, hidden_dim), nn.Tanh()])
        self.decoder = nn.Sequential(*decoder)
        self.out = nn.Linear(hidden_dim, int(np.prod(out_dim)))
        self.out_dim = (c, *out_dim[:2])

    def _emit(self, tape: Tape, z: Act) -> Act:
        for m in self.decoder:
            if isinstance(m, nn.Linear):
                z = tape.linear(z, m, ACT_TANH)
        return tape.linear(z, self.out)

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        h = engine.run_multi(self, self._emit, (_vec(z.float()),))
        h = h.reshape(-1, *self.out_dim)
        return h.squeeze(1) if h.size(1) == 1 else h.permute(0, 2, 3, 1)


class coord_latent(nn.Module):
    """
    The "spatial" part of the rVAE decoder (atomai/nets/ed.py:645-687): fc_coord(2 -> out_dim) +
    fc_latent(latent_dim -> out_dim, no bias) (+ tanh).  Parameter container; executed fused with
    the coordinate transform by engine.Tape.coord_latent.
    """
    def __init__(self, latent_dim: int, out_dim: int, activation: bool = False) -> None:
        super(coord_latent, self).__init__()
        self.fc_coord = nn.Linear(2, out_dim)
        self.fc_latent = nn.Linear(latent_dim, out_dim, bias=False)
        self.activation = nn.Tanh() if activation else None


class rDecoderNet(nn.Module):
    """
    Spatial decoder network (atomai/nets/ed.py:583-642): coord_latent -> num_layers x (Linear +
    tanh) per pixel -> Linear(hidden -> c).

    Two call forms:
      * forward(x_coord, z)  — reference signature; `x_coord` must be the (B, H*W, 2) grid
        produced by imcoordgrid/transform_coordinates.  The rotation angle and shift are
        recovered from the grid (it is an isometry of a known grid), so the fused kernel is used.
      * decode(z, phi=None, dx=None) — native form used by rVAE: coordinates generated on the fly.
    """
    def __init__(self, out_dim: Tuple[int], latent_dim: int, num_layers: int, hidden_dim: int,
                 skip: bool = False) -> None:
        super(rDecoderNet, self).__init__()
        if len(out_dim) == 2:
            c = 1
            self.reshape_ = (out_dim[0], out_dim[1])
        else:
            c = out_dim[-1]
            self.reshape_ = (out_dim[0], out_dim[1], c)
        self.skip = skip
        self.coord_latent = coord_latent(latent_dim, hidden_dim, not skip)
        fc_decoder = []
        for i in range(num_layers):
            fc_decoder.extend([nn.Linear(hidden_dim, hidden_dim), nn.Tanh()])
        self.fc_decoder = nn.Sequential(*fc_decoder)
        self.out = nn.Linear(hidden_dim, c)
        self._c = c

    def _emit(self, tape: Tape, z: Act, phi: Optional[Act] = None, dx: Optional[Act] = None) -> Act:
        h = tape.coord_latent(self.coord_latent, self.reshape_[:2], z, phi, dx,
                              self.coord_latent.activation is not None)
        residual = h
        for m in self.fc_decoder:
            if isinstance(m, nn.Linear):
                h = tape.pointwise(h, m, 1.0, ACT_TANH)
                if self.skip:          # h.add(residual) after every (Linear, Tanh) pair
                    h = tape.add(h, residual)
        return tape.pointwise(h, self.out, 1.0, ACT_LRELU)

    def decode(self, z: torch.Tensor, phi: Optional[torch.Tensor] = None,
               dx: Optional[torch.Tensor] = None) -> torch.Tensor:
        ins = [_vec(z.float())]
        has_phi, has_dx = phi is not None, dx is not None
        if has_phi:
            ins.append(_vec(phi.float().reshape(-1, 1)))
        if has_dx:
            ins.append(_vec(dx.float().reshape(-1, 2)))

        def emit(tape, za, *rest):
            rest = list(rest)
            pa = rest.pop(0) if has_phi else None
            da = rest.pop(0) if has_dx else None
            return self._emit(tape, za, pa, da)
        y = engine.run_multi(self, emit, tuple(ins))                    # (B, H, W, c)
        return y.reshape(y.shape[0], *self.reshape_)

    def forward(self, x_coord: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
        phi, dx = _pose_from_grid(x_coord, self.reshape_[:2])
        return self.decode(z, phi, dx)


def _pose_from_grid(x_coord: torch.Tensor, hw: Tuple[int, int]):
    """Recover (phi, dx) with x_coord = grid @ R(phi) + dx from the first/last grid points
    (grid from imcoordgrid: first row (-1, 1), last row (1, -1); atomai/utils/coords.py:47-83)."""
    p0, p1 = x_coord[:, 0, :], x_coord[:, -1, :]
    dx = 0.5 * (p0 + p1)                                 # grid is symmetric: g0 = -g1
    v = p0 - dx                                          # = (-1, 1) @ R = (-c - s, -s + c)
    c = 0.5 * (v[:, 1] - v[:, 0])
    s = -0.5 * (v[:, 0] + v[:, 1])
    return torch.atan2(s, c), dx


def init_imspec_model(in_dim: Tuple[int], out_dim: Tuple[int], latent_dim: int,
                      **kwargs: Union[int, bool]
                      ) -> Tuple[Type[nn.Module], Dict[str, Union[int, bool]]]:
    """Initializes ImSpec model + meta dict (atomai/nets/ed.py:690-722)."""
    nblayers_encoder = kwargs.get("nblayers_encoder", 3)
    nblayers_decoder = kwargs.get("nblayers_decoder", 4)
    nbfilters_encoder = kwargs.get("nbfilters_encoder", 64)
    nbfilters_decoder = kwargs.get("nbfilters_decoder", 64)
    batch_norm = kwargs.get("batch_norm", True)
    encoder_downsampling = kwargs.get("encoder_downsampling", 0)
    decoder_upsampling = kwargs.get("decoder_upsampling", False)
    net = SignalED(in_dim, out_dim, latent_dim, nblayers_encoder, nblayers_decoder,
                   nbfilters_encoder, nbfilters_decoder, batch_norm, encoder_downsampling,
                   decoder_upsampling)
    meta_state_dict = {
        "model_type": "imspec", "in_dim": in_dim, "out_dim": out_dim, "latent_dim": latent_dim,
        "nblayers_encoder": nblayers_encoder, "nblayers_decoder": nblayers_decoder,
        "nbfilters_encoder": nbfilters_encoder, "nbfilters_decoder": nbfilters_decoder,
        "batchnorm": batch_norm, "encoder_downsampling": encoder_downsampling,
        "decoder_upsampling": decoder_upsampling
    }
    return net, meta_state_dict


def init_VAE_nets(in_dim: Tuple[int], latent_dim: int, coord: int = 0,
                  discrete_dim: Optional[List] = None, nb_classes: int = 0, **kwargs
                  ) -> Tuple[Type[nn.Module], Type[nn.Module], Dict[str, Union[int, bool]]]:
    """Initializes encoder and decoder for VAE + meta dict (atomai/nets/ed.py:725-790).  With
    `discrete_dim` the encoder gets one head per discrete latent and the decoder takes
    latent_dim + sum(discrete_dim) inputs (class conditioning is then off)."""
    conv_e = kwargs.get("conv_encoder", False)
    conv_d = kwargs.get("conv_decoder", False) if not coord else None
    numlayers_e = kwargs.get("numlayers_encoder", 2)
    numlayers_d = kwargs.get("numlayers_decoder", 2)
    numhidden_e = kwargs.get("numhidden_encoder", 128)
    numhidden_d = kwargs.get("numhidden_decoder", 128)
    skip = kwargs.get("skip", False)
    sigmoid_out = kwargs.get("sigmoid_out", False)
    softplus_out = kwargs.get("softplus_out")
    discrete_dim_ = sum(discrete_dim) if discrete_dim else 0
    nb_classes_ = nb_classes if discrete_dim_ == 0 else 0
    if not coord:
        dnet = convDecoderNet if conv_d else fcDecoderNet
        decoder_net = dnet(in_dim, latent_dim + discrete_dim_ + nb_classes_, numlayers_d, numhidden_d)
    else:
        decoder_net = rDecoderNet(in_dim, latent_dim + discrete_dim_ + nb_classes_, numlayers_d,
                                  numhidden_d, skip)
    if not discrete_dim:
        enet = convEncoderNet if conv_e else fcEncoderNet
        encoder_net = enet(in_dim, latent_dim + coord, numlayers_e, numhidden_e,
                           softplus_out=softplus_out)
    else:
        enet = jconvEncoderNet if conv_e else jfcEncoderNet
        encoder_net = enet(in_dim, latent_dim + coord, discrete_dim, numlayers_e, numhidden_e,
                           softplus_out=softplus_out)
    meta_state_dict = {
        "model_type": "vae", "in_dim": in_dim, "latent_dim": latent_dim, "coord": coord,
        "conv_encoder": conv_e, "numlayers_encoder": numlayers_e,
        "numlayers_decoder": numlayers_d, "numhidden_encoder": numhidden_e,
        "numhidden_decoder": numhidden_d, "skip": skip, "nb_classes": nb_classes,
        "discrete_dim": discrete_dim, "sigmoid_out": sigmoid_out, "softplus_out": softplus_out
    }
    if not coord:
        meta_state_dict["conv_decoder"] = conv_d
    return encoder_net, decoder_net, meta_state_dict
