"""
Denoising autoencoder network with the reference's module tree and state_dict keys
(atomai/models/denoiser.py:83-130: `nn.Sequential(encoder, decoder)`), executed as one native
sm_90a graph per call (see atomai_b200/engine.py).
"""
from typing import List

import torch
import torch.nn as nn

from .. import engine
from ..engine import Act, Tape
from .blocks import ConvBlock, UpsampleBlock


class DenoisingAutoencoderNet(nn.Sequential):
    """
    encoder: ConvBlock, MaxPool2d(2, 2), ConvBlock, ..., ConvBlock (no pool after the last block);
    decoder: ConvBlock, [UpsampleBlock(C -> C), ConvBlock] ..., Conv2d(C, 1, 1).
    Children, their order and the state_dict keys (`0.0.block.0.weight`, `1.1.conv.weight`,
    `1.7.weight`, ...) are those of the reference's `_build_autoencoder`; the parameter-free
    MaxPool2d entries keep their indices.
    """
    def __init__(self,
                 encoder_filters: List[int] = (8, 16, 32, 64),
                 decoder_filters: List[int] = (64, 32, 16, 8),
                 encoder_layers: List[int] = (1, 2, 2, 2),
                 decoder_layers: List[int] = (2, 2, 2, 1),
                 batch_norm: bool = False,
                 upsampling_mode: str = "nearest") -> None:
        encoder, in_channels = [], 1
        for i, (filters, layers) in enumerate(zip(encoder_filters, encoder_layers)):
            encoder.append(ConvBlock(2, layers, in_channels, filters, batch_norm=batch_norm))
            if i < len(encoder_filters) - 1:
                encoder.append(nn.MaxPool2d(2, 2))
            in_channels = filters
        decoder = []
        for i, (filters, layers) in enumerate(zip(decoder_filters, decoder_layers)):
            if i > 0:
                decoder.append(UpsampleBlock(2, in_channels, in_channels, mode=upsampling_mode))
            decoder.append(ConvBlock(2, layers, in_channels, filters, batch_norm=batch_norm))
            in_channels = filters
        decoder.append(nn.Conv2d(in_channels, 1, 1))
        super(DenoisingAutoencoderNet, self).__init__(nn.Sequential(*encoder), nn.Sequential(*decoder))

    @property
    def size_multiple(self) -> int:
        """Input height and width must be multiples of this (one 2x2 max-pool per encoder level)."""
        return 2 ** sum(isinstance(m, nn.MaxPool2d) for m in self[0])

    def _emit(self, tape: Tape, x: Act) -> Act:
        for m in (*self[0], *self[1]):
            if isinstance(m, nn.MaxPool2d):
                x = tape.pool(x)
            elif isinstance(m, (ConvBlock, UpsampleBlock)):
                x = m._emit(tape, x)
            else:                       # output layer: 1x1 convolution, no activation
                x = tape.conv(x, m, None, 1.0)
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        k = self.size_multiple
        if x.dim() == 4 and (x.shape[2] % k or x.shape[3] % k):
            raise ValueError(
                f"DenoisingAutoencoder input height and width must be divisible by {k} "
                f"(one 2x2 max-pool per encoder level), got {tuple(x.shape[2:])}")
        return engine.run(self, x)
