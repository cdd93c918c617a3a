"""
Customized NN blocks, same constructor signatures, module tree and state_dict keys as the
reference (atomai/nets/blocks.py:17-132, 257-329), executed by hand-written sm_90a kernels.

The torch sub-modules (nn.Conv2d, nn.LeakyReLU, nn.BatchNorm2d inside `self.block` /
`self.atrous_module`, `self.conv`) are parameter containers only: `forward` never calls them.
It hands the block to the native tape (atomai_b200/engine.py), which fuses bias + LeakyReLU +
BatchNorm statistics into the convolution epilogue and defers the BatchNorm affine, max-pooling
and channel concatenation to the loader of the consuming convolution.
"""
from typing import List, Sequence, Tuple, Union

import torch
import torch.nn as nn

from .. import engine
from ..engine import Act, Tape


def _parse_layers(seq: nn.Sequential) -> List[Tuple[nn.Module, float, nn.Module, float]]:
    """nn.Sequential of [conv, (dropout), lrelu, (bn)] groups -> [(conv, slope, bn|None, p_drop)]."""
    layers, cur = [], None
    for m in seq:
        if isinstance(m, (nn.Conv2d, nn.Conv1d)):
            if cur is not None:
                layers.append(tuple(cur))
            cur = [m, 1.0, None, 0.0]
        elif isinstance(m, nn.LeakyReLU):
            cur[1] = float(m.negative_slope)
        elif isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
            cur[2] = m
        elif isinstance(m, nn.Dropout):
            cur[3] = float(m.p)
        else:
            raise NotImplementedError(f"unsupported layer in block: {type(m).__name__}")
    if cur is not None:
        layers.append(tuple(cur))
    return layers



class ConvBlock(nn.Module):
    """
    Creates block of layers each consisting of convolution operation,
    leaky relu and (optionally) dropout and batch normalization

    Args: see atomai/nets/blocks.py:17-52 (identical signature).
    """
    def __init__(self,
                 ndim: int, nb_layers: int,
                 input_channels: int, output_channels: int,
                 kernel_size: Union[Tuple[int], int] = 3,
                 stride: Union[Tuple[int], int] = 1,
                 padding: Union[Tuple[int], int] = 1,
                 batch_norm: bool = False, lrelu_a: float = 0.01,
                 dropout_: float = 0) -> None:
        super(ConvBlock, self).__init__()
        if not 0 < ndim < 3:
            raise AssertionError("ndim must be equal to 1 or 2")
        conv = nn.Conv2d if ndim == 2 else nn.Conv1d
        block = []
        for idx in range(nb_layers):
            input_channels = output_channels if idx > 0 else input_channels
            block.append(conv(input_channels, output_channels, kernel_size=kernel_size,
                              stride=stride, padding=padding))
            if dropout_ > 0:
                block.append(nn.Dropout(dropout_))
            block.append(nn.LeakyReLU(negative_slope=lrelu_a))
            if batch_norm:
                block.append(nn.BatchNorm2d(output_channels) if ndim == 2
                             else nn.BatchNorm1d(output_channels))
        self.block = nn.Sequential(*block)
        self._squeeze_h = ndim == 1

    def _emit(self, tape: Tape, x: Union[Act, Sequence[Act]]) -> Act:
        for conv, slope, bn, p_drop in _parse_layers(self.block):
            x = tape.conv(x, conv, bn, slope, p_drop=p_drop)
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class UpsampleBlock(nn.Module):
    """
    Defines upsampling block performed using bilinear
    or nearest-neigbor interpolation followed by 1-by-1 convolution
    (atomai/nets/blocks.py:86-132).  The 1x1 convolution is executed BEFORE the interpolation
    (4x fewer FLOPs and bytes; both are linear and the interpolation weights sum to one, so the
    result differs from the reference only by fp32 re-association, SURVEY.md Appendix C).
    """
    def __init__(self,
                 ndim: int,
                 input_channels: int,
                 output_channels: int,
                 scale_factor: int = 2,
                 mode: str = "bilinear") -> None:
        super(UpsampleBlock, self).__init__()
        if not any([mode == 'bilinear', mode == 'nearest']):
            raise NotImplementedError(
                "use 'bilinear' or 'nearest' for upsampling mode")
        if not 0 < ndim < 3:
            raise AssertionError("ndim must be equal to 1 or 2")
        conv = nn.Conv2d if ndim == 2 else nn.Conv1d
        self.scale_factor = scale_factor
        self.mode = mode if ndim == 2 else "nearest"
        self.conv = conv(input_channels, output_channels, kernel_size=1, stride=1, padding=0)
        self._squeeze_h = ndim == 1
        self._ndim = ndim

    def _emit(self, tape: Tape, x: Act) -> Act:
        if self.scale_factor != 2 or self._ndim != 2:
            raise NotImplementedError("native UpsampleBlock supports 2-D, scale_factor=2")
        low = tape.conv(x, self.conv, None, 1.0)
        return tape.upsample(low, self.mode)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class ResBlock(nn.Module):
    """
    Builds a residual block: 1x1 conv -> [3x3 conv -> BN -> LeakyReLU -> 3x3 conv -> BN] + skip ->
    LeakyReLU (atomai/nets/blocks.py:135-214; identical signature and parameter names).  Natively:
    three wgmma convolutions with the BatchNorm statistics in their epilogues, and the
    BN-affine + residual add + LeakyReLU tails as one HBM pass each (csrc/resnet.cu).
    """
    def __init__(self,
                 ndim: int,
                 input_channels: int,
                 output_channels: int,
                 kernel_size: Union[Tuple[int], int] = 3,
                 stride: Union[Tuple[int], int] = 1,
                 padding: Union[Tuple[int], int] = 1,
                 batch_norm: bool = True,
                 lrelu_a: float = 0.01) -> None:
        super(ResBlock, self).__init__()
        if not 0 < ndim < 3:
            raise AssertionError("ndim must be equal to 1 or 2")
        conv = nn.Conv2d if ndim == 2 else nn.Conv1d
        self.lrelu_a = lrelu_a
        self.batch_norm = batch_norm
        self.c0 = conv(input_channels, output_channels, kernel_size=1, stride=1, padding=0)
        self.c1 = conv(output_channels, output_channels, kernel_size=3, stride=1, padding=1)
        self.c2 = conv(output_channels, output_channels, kernel_size=3, stride=1, padding=1)
        if batch_norm:
            bn = nn.BatchNorm2d if ndim == 2 else nn.BatchNorm1d
            self.bn1 = bn(output_channels)
            self.bn2 = bn(output_channels)
        self._squeeze_h = ndim == 1

    def _emit(self, tape: Tape, x: Union[Act, Sequence[Act]]) -> Act:
        a = float(self.lrelu_a)
        if not a > 0:
            raise NotImplementedError("native ResBlock needs a LeakyReLU slope > 0")
        x0 = tape.conv(x, self.c0, None, 1.0)                       # residual
        if self.batch_norm:
            h = tape.bn_res_act(tape.conv(x0, self.c1, self.bn1, 1.0), None, a)
            return tape.bn_res_act(tape.conv(h, self.c2, self.bn2, 1.0), x0, a)
        h = tape.conv(x0, self.c1, None, a)                          # fused LeakyReLU epilogue
        return tape.bn_res_act(tape.conv(h, self.c2, None, 1.0), x0, a)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class ResModule(nn.Module):
    """
    Stitches multiple convolutional blocks with residual connections together
    (atomai/nets/blocks.py:217-254).
    """
    def __init__(self,
                 ndim: int,
                 res_depth: int,
                 input_channels: int,
                 output_channels: int,
                 batch_norm: bool = True,
                 lrelu_a: float = 0.01) -> None:
        super(ResModule, self).__init__()
        res_module = []
        for i in range(res_depth):
            input_channels = output_channels if i > 0 else input_channels
            res_module.append(
                ResBlock(ndim, input_channels, output_channels,
                         lrelu_a=lrelu_a, batch_norm=batch_norm))
        self.res_module = nn.Sequential(*res_module)
        self._squeeze_h = ndim == 1

    def _emit(self, tape: Tape, x: Union[Act, Sequence[Act]]) -> Act:
        for blk in self.res_module:
            x = blk._emit(tape, x)
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class DilatedBlock(nn.Module):
    """
    Creates a "cascade" with dilated convolutional layers (aka atrous convolutions);
    the output is the sum of the outputs of EVERY sub-module of the cascade
    (atomai/nets/blocks.py:257-329).
    """
    def __init__(self, ndim: int, input_channels: int, output_channels: int,
                 dilation_values: List[int], padding_values: List[int],
                 kernel_size: Union[Tuple[int], int] = 3,
                 stride: Union[Tuple[int], int] = 1, lrelu_a: float = 0.01,
                 batch_norm: bool = False, dropout_: float = 0) -> None:
        super(DilatedBlock, self).__init__()
        if not 0 < ndim < 3:
            raise AssertionError("ndim must be equal to 1 or 2")
        conv = nn.Conv2d if ndim == 2 else nn.Conv1d
        atrous_module = []
        for idx, (dil, pad) in enumerate(zip(dilation_values, padding_values)):
            input_channels = output_channels if idx > 0 else input_channels
            atrous_module.append(conv(input_channels, output_channels, kernel_size=kernel_size,
                                      stride=stride, padding=pad, dilation=dil, bias=True))
            if dropout_ > 0:
                atrous_module.append(nn.Dropout(dropout_))
            atrous_module.append(nn.LeakyReLU(negative_slope=lrelu_a))
            if batch_norm:
                atrous_module.append(nn.BatchNorm2d(output_channels) if ndim == 2
                                     else nn.BatchNorm1d(output_channels))
        self.atrous_module = nn.Sequential(*atrous_module)
        self._squeeze_h = ndim == 1

    def _emit(self, tape: Tape, x: Act) -> Act:
        outs, slope0 = [], None
        for conv, slope, bn, p_drop in _parse_layers(self.atrous_module):
            if p_drop > 0 and self.training:
                raise NotImplementedError(
                    "DilatedBlock with training-mode dropout: the reference sums the outputs of "
                    "every sub-module including the Dropout's (blocks.py:321-329); not implemented")
            x = tape.conv(x, conv, bn, slope)
            outs.append(x)
            slope0 = slope if slope0 is None else slope0
        return tape.dilated_sum(outs, slope0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)
