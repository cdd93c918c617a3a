"""
Fully convolutional neural networks — Unet and dilnet with the reference's constructor
signatures, module names and checkpoint layout (atomai/nets/fcnn.py:18-226, 379-442), executed
as one native sm_90a graph per call (see atomai_b200/engine.py).

ResHedNet / SegResNet (ResBlock based, atomai/nets/fcnn.py:229-376) run on the same native tape.
"""
from typing import List, Type, Union

import torch
import torch.nn as nn

from .. import engine
from ..engine import Act, Tape
from .blocks import ConvBlock, DilatedBlock, ResModule, UpsampleBlock


class Unet(nn.Module):
    """
    Builds a fully convolutional Unet-like neural network model
    (arguments as in atomai/nets/fcnn.py:18-57).
    """
    def __init__(self,
                 nb_classes: int = 1,
                 nb_filters: int = 16,
                 dropout: bool = False,
                 batch_norm: bool = True,
                 upsampling_mode: str = "bilinear",
                 with_dilation: bool = False,
                 **kwargs: List[int]) -> None:
        super(Unet, self).__init__()
        nbl = kwargs.get("layers", [1, 2, 2, 3])
        dilation_values = torch.arange(2, 2*nbl[-1]+1, 2).tolist()
        padding_values = dilation_values.copy()
        dropout_vals = [.1, .2, .1] if dropout else [0, 0, 0]
        self.c1 = ConvBlock(2, nbl[0], 1, nb_filters, batch_norm=batch_norm)
        self.c2 = ConvBlock(2, nbl[1], nb_filters, nb_filters*2, batch_norm=batch_norm)
        self.c3 = ConvBlock(2, nbl[2], nb_filters*2, nb_filters*4, batch_norm=batch_norm,
                            dropout_=dropout_vals[0])
        if with_dilation:
            self.bn = DilatedBlock(2, nb_filters*4, nb_filters*8,
                                   dilation_values=dilation_values,
                                   padding_values=padding_values,
                                   batch_norm=batch_norm, dropout_=dropout_vals[1])
        else:
            self.bn = ConvBlock(2, nbl[3], nb_filters*4, nb_filters*8, batch_norm=batch_norm,
                                dropout_=dropout_vals[1])
        self.upsample_block1 = UpsampleBlock(2, nb_filters*8, nb_filters*4, mode=upsampling_mode)
        self.c4 = ConvBlock(2, nbl[2], nb_filters*8, nb_filters*4, batch_norm=batch_norm,
                            dropout_=dropout_vals[2])
        self.upsample_block2 = UpsampleBlock(2, nb_filters*4, nb_filters*2, mode=upsampling_mode)
        self.c5 = ConvBlock(2, nbl[1], nb_filters*4, nb_filters*2, batch_norm=batch_norm)
        self.upsample_block3 = UpsampleBlock(2, nb_filters*2, nb_filters, mode=upsampling_mode)
        self.c6 = ConvBlock(2, nbl[0], nb_filters*2, nb_filters, batch_norm=batch_norm)
        self.px = nn.Conv2d(nb_filters, nb_classes, 1, 1, 0)

    def _emit(self, tape: Tape, x: Act) -> Act:
        # Contracting path (pooling is deferred to the consumer's loader)
        c1 = self.c1._emit(tape, x)
        c2 = self.c2._emit(tape, tape.pool(c1))
        c3 = self.c3._emit(tape, tape.pool(c2))
        # Bottleneck layer
        bn = self.bn._emit(tape, tape.pool(c3))
        # Expanding path: torch.cat([skip, up], 1) becomes a two-source convolution
        u3 = self.upsample_block1._emit(tape, bn)
        u3 = self.c4._emit(tape, [c3, u3])
        u2 = self.upsample_block2._emit(tape, u3)
        u2 = self.c5._emit(tape, [c2, u2])
        u1 = self.upsample_block3._emit(tape, u2)
        u1 = self.c6._emit(tape, [c1, u1])
        # Final layer used for pixel-wise convolution
        return tape.conv(u1, self.px, None, 1.0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class dilnet(nn.Module):
    """
    Builds a fully convolutional neural network model by utilizing a combination of regular and
    dilated convolutions (arguments as in atomai/nets/fcnn.py:145-175).
    """
    def __init__(self,
                 nb_classes: int = 1,
                 nb_filters: int = 25,
                 dropout: bool = False,
                 batch_norm: bool = True,
                 upsampling_mode: str = "bilinear",
                 **kwargs: List[int]) -> None:
        super(dilnet, self).__init__()
        nbl = kwargs.get("layers", [3, 3, 3, 3])
        dilation_values_1 = torch.arange(2, 2*nbl[1]+1, 2).tolist()
        padding_values_1 = dilation_values_1.copy()
        dilation_values_2 = torch.arange(2, 2*nbl[2]+1, 2).tolist()
        padding_values_2 = dilation_values_2.copy()
        dropout_vals = [.3, .3] if dropout else [0, 0]
        self.c1 = ConvBlock(2, nbl[0], 1, nb_filters, batch_norm=batch_norm)
        self.at1 = DilatedBlock(2, nb_filters, nb_filters*2,
                                dilation_values=dilation_values_1,
                                padding_values=padding_values_1,
                                batch_norm=batch_norm, dropout_=dropout_vals[0])
        self.at2 = DilatedBlock(2, nb_filters*2, nb_filters*2,
                                dilation_values=dilation_values_2,
                                padding_values=padding_values_2,
                                batch_norm=batch_norm, dropout_=dropout_vals[1])
        self.up1 = UpsampleBlock(2, nb_filters*2, nb_filters, mode=upsampling_mode)
        self.c2 = ConvBlock(2, nbl[3], nb_filters*2, nb_filters, batch_norm=batch_norm)
        self.px = nn.Conv2d(nb_filters, nb_classes, 1, 1, 0)

    def _emit(self, tape: Tape, x: Act) -> Act:
        c1 = self.c1._emit(tape, x)
        at1 = self.at1._emit(tape, tape.pool(c1))
        at2 = self.at2._emit(tape, at1)
        u1 = self.up1._emit(tape, at2)
        u1 = self.c2._emit(tape, [c1, u1])
        return tape.conv(u1, self.px, None, 1.0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class ResHedNet(nn.Module):
    """
    Holistically nested edge detector with residual connections in each block
    (arguments, module names and state_dict keys as in atomai/nets/fcnn.py:229-296).
    """
    def __init__(self,
                 nb_classes: int = 1,
                 nb_filters: int = 64,
                 upsampling_mode: str = "bilinear",
                 **kwargs: List[int]) -> None:
        super(ResHedNet, self).__init__()
        nbl = kwargs.get("layers", [3, 4, 5])
        self.upsample = upsampling_mode
        self.net1 = ResModule(2, nbl[0], 1, nb_filters, True)
        self.net2 = nn.Sequential(
            nn.MaxPool2d(2, 2),
            ResModule(2, nbl[1], nb_filters, 2*nb_filters, True)
        )
        self.net3 = nn.Sequential(
            nn.MaxPool2d(2, 2),
            ResModule(2, nbl[2], 2*nb_filters, 4*nb_filters, True)
        )
        self.net1score = nn.Sequential(
            nn.Conv2d(nb_filters, nb_classes, 1, 1, 0),
            nn.BatchNorm2d(nb_classes)
        )
        self.net2score = nn.Sequential(
            nn.Conv2d(2*nb_filters, nb_classes, 1, 1, 0),
            nn.BatchNorm2d(nb_classes)
        )
        self.net3score = nn.Sequential(
            nn.Conv2d(4*nb_filters, nb_classes, 1, 1, 0),
            nn.BatchNorm2d(nb_classes)
        )
        self.out = torch.nn.Conv2d(3*nb_classes, nb_classes, 1, 1, 0)

    def _emit(self, tape: Tape, x: Act) -> Act:
        n1 = self.net1._emit(tape, x)
        n2 = self.net2[1]._emit(tape, tape.pool(n1))
        n3 = self.net3[1]._emit(tape, tape.pool(n2))
        # side outputs: 1x1 conv -> BatchNorm (no activation), brought to the input size
        s1 = tape.conv(n1, self.net1score[0], self.net1score[1], 1.0)
        s2 = tape.resize(tape.conv(n2, self.net2score[0], self.net2score[1], 1.0), 2, self.upsample)
        s3 = tape.resize(tape.conv(n3, self.net3score[0], self.net3score[1], 1.0), 4, self.upsample)
        return tape.conv(tape.cat([s1, s2, s3]), self.out, None, 1.0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


class SegResNet(nn.Module):
    """
    Builds a fully convolutional neural network based on SegNet architecture
    with residual blocks for semantic segmentation
    (arguments, module names and state_dict keys as in atomai/nets/fcnn.py:299-376).
    """
    def __init__(self,
                 nb_classes: int = 1,
                 nb_filters: int = 32,
                 batch_norm: bool = True,
                 upsampling_mode: str = "bilinear",
                 **kwargs: List[int]) -> None:
        super(SegResNet, self).__init__()
        nbl = kwargs.get("layers", [2, 2, 2])
        self.c1 = ConvBlock(2, 1, 1, nb_filters, batch_norm=batch_norm)
        self.c2 = ResModule(2, nbl[0], nb_filters, nb_filters*2, batch_norm=batch_norm)
        self.bn = ResModule(2, nbl[1], nb_filters*2, nb_filters*4, batch_norm=batch_norm)
        self.upsample_block1 = UpsampleBlock(2, nb_filters*4, nb_filters*2, 2, upsampling_mode)
        self.c3 = ResModule(2, nbl[2], nb_filters*4, nb_filters*2, batch_norm=batch_norm)
        self.upsample_block2 = UpsampleBlock(2, nb_filters*2, nb_filters, 2, upsampling_mode)
        self.c4 = ConvBlock(2, 1, nb_filters*2, nb_filters, batch_norm=batch_norm)
        self.px = nn.Conv2d(nb_filters, nb_classes, 1, 1, 0)

    def _emit(self, tape: Tape, x: Act) -> Act:
        c1 = self.c1._emit(tape, x)
        c2 = self.c2._emit(tape, tape.pool(c1))
        bn = self.bn._emit(tape, tape.pool(c2))
        u2 = self.upsample_block1._emit(tape, bn)
        u2 = self.c3._emit(tape, [c2, u2])
        u1 = self.upsample_block2._emit(tape, u2)
        u1 = self.c4._emit(tape, [c1, u1])
        return tape.conv(u1, self.px, None, 1.0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return engine.run(self, x)


def init_fcnn_model(model: Union[Type[nn.Module], str],
                    nb_classes: int, **kwargs: [bool, int, List]
                    ) -> Type[nn.Module]:
    """
    Initializes a fully convolutional neural network; returns (net, meta_state_dict) with the
    reference's metadata keys (atomai/nets/fcnn.py:379-442).
    """
    if not isinstance(model, str) and hasattr(model, "state_dict"):
        meta_state_dict = {
            'model_type': 'Seg', model: 'custom', 'nb_classes': nb_classes}
        return model, meta_state_dict
    batch_norm = kwargs.get('batch_norm', True)
    dropout = kwargs.get('dropout', False)
    upsampling = kwargs.get('upsampling', "bilinear")
    meta_state_dict = {
        'model_type': 'seg',
        'model': model,
        'nb_classes': nb_classes,
        'batch_norm': batch_norm,
        'dropout': dropout,
        'upsampling': upsampling,
    }
    if isinstance(model, str) and model == 'Unet':
        with_dilation = kwargs.get('with_dilation', False)
        nb_filters = kwargs.get('nb_filters', 16)
        layers = kwargs.get("layers", [1, 2, 2, 3])
        net = Unet(nb_classes, nb_filters, dropout, batch_norm, upsampling, with_dilation,
                   layers=layers)
        meta_state_dict["with_dilation"] = with_dilation
    elif isinstance(model, str) and model == 'dilnet':
        nb_filters = kwargs.get('nb_filters', 25)
        layers = kwargs.get("layers", [1, 3, 3, 1])
        net = dilnet(nb_classes, nb_filters, dropout, batch_norm, upsampling, layers=layers)
    elif isinstance(model, str) and model == 'SegResNet':
        nb_filters = kwargs.get('nb_filters', 32)
        layers = kwargs.get("layers", [2, 2, 2])
        net = SegResNet(nb_classes, nb_filters, batch_norm, upsampling, layers=layers)
    elif isinstance(model, str) and model == 'ResHedNet':
        nb_filters = kwargs.get('nb_filters', 64)
        layers = kwargs.get("layers", [3, 4, 5])
        net = ResHedNet(nb_classes, nb_filters, upsampling, layers=layers)
    else:
        raise NotImplementedError(
            "Currently implemented models are 'Unet', 'dilnet', SegResNet', and 'ResHedNet'"
        )
    if model in ["ResHedNet", "SegResNet"]:
        meta_state_dict["dropout"] = None          # (atomai/nets/fcnn.py:436-439, quirk kept)
    meta_state_dict["nb_filters"] = nb_filters
    meta_state_dict["layers"] = layers
    return net, meta_state_dict
