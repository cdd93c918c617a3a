"""
TEST INFRASTRUCTURE — functional restatement (plain torch ops, any dtype; the tests use float64)
of the reference's DenoisingAutoencoder network (atomai/models/denoiser.py:83-130): forward in
eval or train mode, MSE loss, and one BaseTrainer.train_step with Adam.  The backward is torch
autograd over these expressions.  Pinned to the reference goldens in tests/test_dae.py
(tests/golden/make_golden_dae.py); the GPU tests use it for shapes the goldens do not cover.

The model is (cfg, {reference state_dict key -> tensor}); cfg holds the constructor arguments
encoder_filters, decoder_filters, encoder_layers, decoder_layers, use_batch_norm, upsampling_mode.
"""
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from .nets_ref import SD, _conv, adam_step, conv_block, upsample_block

DEFAULTS = dict(encoder_filters=[8, 16, 32, 64], decoder_filters=[64, 32, 16, 8],
                encoder_layers=[1, 2, 2, 2], decoder_layers=[2, 2, 2, 1],
                use_batch_norm=False, upsampling_mode="nearest")


def dae_forward(x, sd: SD, cfg: dict, training: bool = False, new_stats: Optional[dict] = None):
    """nn.Sequential(encoder, decoder) of _build_autoencoder: encoder ConvBlocks with a 2x2
    max-pool after every block but the last; decoder ConvBlocks, each after the first preceded by
    UpsampleBlock(C -> C) (interpolate, then 1x1 conv); a final 1x1 Conv2d(C, 1)."""
    c = dict(DEFAULTS, **cfg)
    kw = dict(batch_norm=c["use_batch_norm"], training=training, new_stats=new_stats)
    i = 0
    nenc = len(c["encoder_filters"])
    for lvl, (_, layers) in enumerate(zip(c["encoder_filters"], c["encoder_layers"])):
        x = conv_block(x, sd, f"0.{i}", layers, **kw)
        i += 1
        if lvl < nenc - 1:
            x = F.max_pool2d(x, 2, 2)
            i += 1
    j = 0
    for lvl, (_, layers) in enumerate(zip(c["decoder_filters"], c["decoder_layers"])):
        if lvl > 0:
            x = upsample_block(x, sd, f"1.{j}", c["upsampling_mode"])
            j += 1
        x = conv_block(x, sd, f"1.{j}", layers, **kw)
        j += 1
    return _conv(x, sd, f"1.{j}")


def dae_train_step(x, y, sd: SD, cfg: dict, opt_state: dict, lr=1e-3) -> Tuple[float, SD]:
    """Train-mode forward, MSE loss, backward, Adam (BaseTrainer.train_step with loss='mse').
    Mutates sd (weights + BatchNorm running statistics) and opt_state; returns (loss, grads)."""
    names = [k for k in sd if sd[k].dtype.is_floating_point and "running_" not in k]
    leaves = {k: sd[k].detach().clone().requires_grad_(True) for k in names}
    work = dict(sd)
    work.update(leaves)
    new_stats = {}
    loss = F.mse_loss(dae_forward(x, work, cfg, training=True, new_stats=new_stats), y)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names])
    opt_state["step"] = opt_state.get("step", 0) + 1
    if "m" not in opt_state:
        opt_state["m"] = [torch.zeros_like(sd[k]) for k in names]
        opt_state["v"] = [torch.zeros_like(sd[k]) for k in names]
    with torch.no_grad():
        adam_step([sd[k] for k in names], list(grads), opt_state["m"], opt_state["v"],
                  opt_state["step"], lr)
        for k, t in new_stats.items():
            sd[k].copy_(t)
        for k in sd:
            if k.endswith("num_batches_tracked"):
                sd[k] += 1
    return float(loss), {k: g for k, g in zip(names, grads)}
