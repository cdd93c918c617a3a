"""
Regressor and classifier networks with a MobileNetV2 backbone (atomai/nets/reg_cls.py:16-150,
atomai/nets/blocks.py:332-399), executed as one native sm_90a graph per call (atomai_b200/mbv2.py).

The module tree is built from plain nn.Conv2d / nn.BatchNorm2d / nn.ReLU6 / nn.Sequential, without
torchvision, and gives the reference's state_dict keys, shapes and order
(`backbone.backbone_layers.0.0.weight` ... `backbone.backbone_layers.18.1.num_batches_tracked`,
then `output_layer.weight` or `output_layer.0.weight`), so reference checkpoints load unchanged.
Its initialisation draws from torch's generator in the order torchvision's mobilenet_v2 and the
reference's stem replacement do, so the same seed gives the same weights.
"""
import torch
import torch.nn as nn

from .. import engine, mbv2

# (expansion t, output channels c, repeats n, first stride s) of MobileNetV2
_SETTINGS = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1),
             (6, 160, 3, 2), (6, 320, 1, 1))
_LAST = 1280


def _conv_bn_relu6(cin: int, cout: int, k: int, stride: int = 1, groups: int = 1) -> nn.Sequential:
    return nn.Sequential(nn.Conv2d(cin, cout, k, stride, (k - 1) // 2, groups=groups, bias=False),
                         nn.BatchNorm2d(cout), nn.ReLU6(inplace=True))


class InvertedResidual(nn.Module):
    """[1x1 expand ->] depthwise 3x3 (stride s) -> linear 1x1 project; adds the input when s = 1
    and the widths match.  `conv` holds the layers under the reference's keys."""
    def __init__(self, cin: int, cout: int, stride: int, expand_ratio: int) -> None:
        super(InvertedResidual, self).__init__()
        self.stride = stride
        hidden = cin * expand_ratio
        self.use_res_connect = stride == 1 and cin == cout
        layers = []
        if expand_ratio != 1:
            layers.append(_conv_bn_relu6(cin, hidden, 1))
        layers += [_conv_bn_relu6(hidden, hidden, 3, stride, groups=hidden),
                   nn.Conv2d(hidden, cout, 1, 1, 0, bias=False), nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*layers)
        self.out_channels = cout

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        raise RuntimeError("InvertedResidual runs inside RegressorNet / ClassifierNet")

    def _emit(self, tape, x):
        mods = list(self.conv)
        h = x
        if len(mods) == 4:
            exp = mods.pop(0)
            h = mbv2.pointwise(tape, h, exp[0], exp[1], relu6=True)
        dw, proj, bn = mods
        h = mbv2.conv3x3(tape, h, dw[0], dw[1])
        h = mbv2.pointwise(tape, h, proj, bn, relu6=False)
        if self.use_res_connect:
            h = tape.bn_res_act(h, x, 1.0)      # BatchNorm(h) + x (slope 1: no activation)
        return h


class CustomBackbone(nn.Module):
    """MobileNetV2 feature extractor + AdaptiveAvgPool2d(1) (atomai/nets/blocks.py:332-399).
    Only backbone_type='mobilenet' runs natively."""
    def __init__(self, input_channels: int, backbone_type: str = "mobilenet") -> None:
        super(CustomBackbone, self).__init__()
        if backbone_type in ("resnet", "vgg"):
            raise NotImplementedError(
                f"backbone_type='{backbone_type}' is not implemented on the native path; "
                "use backbone_type='mobilenet'")
        if backbone_type != "mobilenet":
            raise ValueError("Unsupported backbone_type. Choose 'mobilenet'.")
        # torchvision's mobilenet_v2(): stem for 3 channels, blocks, last layer, classifier head,
        # then its weight initialisation; the reference then swaps in its own stem (blocks.py:378)
        layers = [_conv_bn_relu6(3, 32, 3, 2)]
        cin = 32
        for t, c, n, s in _SETTINGS:
            for i in range(n):
                layers.append(InvertedResidual(cin, c, s if i == 0 else 1, t))
                cin = c
        layers.append(_conv_bn_relu6(cin, _LAST, 1))
        features = nn.Sequential(*layers)
        classifier = nn.Sequential(nn.Dropout(p=0.2), nn.Linear(_LAST, 1000))
        for m in nn.Sequential(features, classifier).modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)
        features[0][0] = nn.Conv2d(input_channels, 32, kernel_size=3, stride=2, padding=1, bias=False)
        self.in_features = _LAST
        self.backbone_layers = features
        self.adaptive_pool = nn.AdaptiveAvgPool2d((1, 1))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        raise RuntimeError("CustomBackbone runs inside RegressorNet / ClassifierNet")

    def _emit(self, tape, x):
        layers = list(self.backbone_layers)
        stem, last = layers[0], layers[-1]
        h = mbv2.conv3x3(tape, x, stem[0], stem[1])
        for blk in layers[1:-1]:
            h = blk._emit(tape, h)
        h = mbv2.pointwise(tape, h, last[0], last[1], relu6=True)
        return mbv2.avgpool(tape, h)


class _RegClsNet(nn.Module):
    def _head(self, tape, x):
        raise NotImplementedError

    def _emit_nhwc(self, tape, x):
        return self._head(tape, self.backbone._emit(tape, x))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.dim() != 4:
            raise ValueError(f"expected (N, C, H, W) input, got shape {tuple(x.shape)}")
        out = engine.run_multi(self, self._emit_nhwc, [engine._to_nhwc(x)],
                               comm=getattr(self, "_comm", None))
        return out.reshape(out.shape[0], out.shape[3])


class RegressorNet(_RegClsNet):
    """MobileNetV2 backbone -> flatten -> Linear(1280, output_size)."""
    def __init__(self, input_channels: int, output_size: int, backbone_type: str = "mobilenet"):
        super(RegressorNet, self).__init__()
        self.backbone = CustomBackbone(input_channels, backbone_type)
        self.output_layer = nn.Linear(self.backbone.in_features, output_size)
        self.flatten = nn.Flatten()

    def _head(self, tape, x):
        return mbv2.linear(tape, x, self.output_layer)


class ClassifierNet(_RegClsNet):
    """MobileNetV2 backbone -> flatten -> Linear(1280, num_classes) -> LogSoftmax(dim=1)."""
    def __init__(self, input_channels: int, num_classes: int, backbone_type: str = "resnet"):
        super(ClassifierNet, self).__init__()
        self.backbone = CustomBackbone(input_channels, backbone_type)
        self.output_layer = nn.Sequential(nn.Linear(self.backbone.in_features, num_classes),
                                          nn.LogSoftmax(dim=1))
        self.flatten = nn.Flatten()

    def _head(self, tape, x):
        return mbv2.log_softmax(tape, mbv2.linear(tape, x, self.output_layer[0]))


def init_reg_model(out_dim, backbone_type, input_channels=1, **kwargs):
    """Initializes a regression model with a specified backbone type"""
    net = RegressorNet(input_channels, out_dim, backbone_type)
    meta_state_dict = {
        "model_type": "reg",
        "backbone": backbone_type,
        "in_channels": input_channels,
        "out_dim": out_dim
    }
    return net, meta_state_dict


def init_cls_model(num_classes, backbone_type, input_channels=1, **kwargs):
    """Initializes a classification model with a specified backbone type"""
    net = ClassifierNet(input_channels, num_classes, backbone_type)
    meta_state_dict = {
        "model_type": "cls",
        "backbone": backbone_type,
        "in_channels": input_channels,
        "nb_classes": num_classes
    }
    return net, meta_state_dict
