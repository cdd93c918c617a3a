"""
Restatement of the reference's RegressorNet / ClassifierNet with the MobileNetV2 backbone
(atomai/nets/reg_cls.py:16-84, atomai/nets/blocks.py:332-399 -> torchvision mobilenet_v2) as plain
torch.nn.functional calls on a state_dict, without torchvision.  Runs in any dtype (the tests use
float64 on the CPU and the GPU); pinned to the reference's goldens by tests/test_regcls.py.
"""
import torch
import torch.nn.functional as F

SETTINGS = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1),
            (6, 160, 3, 2), (6, 320, 1, 1))


def _bn(x, sd, pre, training, new_stats):
    rm, rv = sd[pre + ".running_mean"].clone(), sd[pre + ".running_var"].clone()
    y = F.batch_norm(x, rm, rv, sd[pre + ".weight"], sd[pre + ".bias"], training, 0.1, 1e-5)
    if training and new_stats is not None:
        new_stats[pre + ".running_mean"] = rm
        new_stats[pre + ".running_var"] = rv
    return y


def _cbr(x, sd, pre, stride, groups, training, new_stats, relu6=True):
    w = sd[pre + ".0.weight"]
    x = F.conv2d(x, w, None, stride, w.shape[-1] // 2, 1, groups)
    x = _bn(x, sd, pre + ".1", training, new_stats)
    return F.relu6(x) if relu6 else x


def blocks():
    """(index, cin, cout, stride, expand) of the 17 inverted-residual blocks."""
    out, i, cin = [], 1, 32
    for t, c, n, s in SETTINGS:
        for j in range(n):
            out.append((i, cin, c, s if j == 0 else 1, t))
            cin, i = c, i + 1
    return out


def backbone(x, sd, training=True, new_stats=None):
    """(N, C, H, W) -> (N, 1280) pooled features."""
    b = "backbone.backbone_layers."
    h = _cbr(x, sd, b + "0", 2, 1, training, new_stats)
    for i, cin, cout, s, t in blocks():
        pre = f"{b}{i}.conv."
        y, k = h, 0
        if t != 1:
            y = _cbr(y, sd, pre + "0", 1, 1, training, new_stats)
            k = 1
        hidden = cin * t
        y = _cbr(y, sd, f"{pre}{k}", s, hidden, training, new_stats)
        y = F.conv2d(y, sd[f"{pre}{k + 1}.weight"])
        y = _bn(y, sd, f"{pre}{k + 2}", training, new_stats)
        h = h + y if (s == 1 and cin == cout) else y
    h = _cbr(h, sd, b + "18", 1, 1, training, new_stats)
    return F.adaptive_avg_pool2d(h, 1).flatten(1)


def regressor_forward(x, sd, training=True, new_stats=None):
    return F.linear(backbone(x, sd, training, new_stats), sd["output_layer.weight"],
                    sd["output_layer.bias"])


def classifier_forward(x, sd, training=True, new_stats=None):
    z = F.linear(backbone(x, sd, training, new_stats), sd["output_layer.0.weight"],
                 sd["output_layer.0.bias"])
    return F.log_softmax(z, dim=1)


def forward(kind, x, sd, training=True, new_stats=None):
    return (regressor_forward if kind == "reg" else classifier_forward)(x, sd, training, new_stats)


def loss(kind, out, y):
    return F.mse_loss(out, y) if kind == "reg" else F.nll_loss(out, y)
