"""Kernel-level parity through the C ABI (ctypes -> libatomai_b200.so) against plain PyTorch fp32
ops on the same GPU: every export of include/atomai_b200.h the hot path uses, in both math modes,
plus size-independent properties at the BASELINE.json workload size (32 x 512 x 512).

The case library lives in tools/gpu_check1.py (also used for bring-up on the box); thresholds:
  fp32 (exact FFMA kernels)   rel = max|a-ref|/max|ref| <= 5e-6, BN statistics 1e-6
  tf32 (wgmma)                rel <= 1e-3 (TF32 operand rounding, measured 2.6-4.2e-4), stats 5e-4
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu


def _run(group):
    import gpu_check1
    return gpu_check1.run_group(group)


@pytest.mark.parametrize("group,tol,stol", [("simt", 5e-6, 1e-6), ("tc_basic", 1e-3, 5e-4),
                                            ("tc_fused", 1e-3, 5e-4)])
def test_conv_forward(cuda, group, tol, stol):
    """atomai_b200_conv_fwd: conv + bias + LeakyReLU + BN statistics, normalise-on-load, pool-on-load,
    two-source concat, dilation, NCHW head output, ragged sizes — vs F.conv2d / F.leaky_relu."""
    for k, v in _run(group).items():
        assert v["rel"] <= tol, (k, v)
        if "stats_rel" in v:
            assert v["stats_rel"] <= stol, (k, v)


def test_conv_dgrad(cuda):
    """data gradient = the same kernel with AB_WMODE_DGRAD weights, vs autograd."""
    for k, v in _run("tc_dgrad").items():
        assert v["rel"] <= (5e-6 if k.startswith("simt") else 1e-3), (k, v)


@pytest.mark.parametrize("group,tol", [("wgrad_simt", 5e-6), ("wgrad_tc", 1e-3)])
def test_conv_wgrad(cuda, group, tol):
    """atomai_b200_conv_wgrad vs autograd's weight gradient."""
    for k, v in _run(group).items():
        assert v["rel"] <= tol, (k, v)


def test_elementwise_and_optimizer(cuda):
    """BN finalize/affine/backward, pool, upsample, cross-entropy, fused Adam vs torch."""
    for k, v in _run("elementwise").items():
        assert v["rel"] <= 2e-5, (k, v)


def test_linear_and_gram(cuda):
    for k, v in _run("vae").items():
        assert v["rel"] <= 1e-4, (k, v)


def test_full_size_linearity(cuda):
    """BASELINE-size layer (32 x 512 x 512, 16 -> 16): the oracle cannot run here in seconds, so the
    check is a size-independent property — with identity activation and no bias the fused conv is
    linear in its input, and the weight gradient is linear in dy."""
    from atomai_b200 import ops
    from atomai_b200.ops import Source
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(3)
    N, H, W, C = 32, 512, 512, 16
    x1 = torch.randn(N, H, W, C, generator=g).to(dev)
    x2 = torch.randn(N, H, W, C, generator=g).to(dev)
    w = (torch.randn(C, C, 3, 3, generator=g) * 0.1).to(dev)
    outs = []
    for x in (x1, x2, x1 + x2):
        d = ops.conv_desc([Source(x)], N, H, W, C, (3, 3), 1, 1.0, ops.MATH_TF32)
        wp = ops.prep_weights(w, ops.WMODE_FWD, ops.MATH_TF32)
        o = torch.empty(N, H, W, C, device=dev)
        ops.conv_fwd(d, wp, None, o, None)
        outs.append(o)
    err = (outs[0] + outs[1] - outs[2]).abs().max() / outs[2].abs().max()
    assert float(err) <= 2e-3, float(err)
    # border rows must see zero padding: the first output row only uses kernel rows 1, 2
    ref_row = torch.nn.functional.conv2d(x1[:1, :2].permute(0, 3, 1, 2), w[:, :, 1:, :], padding=(0, 1))
    got_row = outs[0][:1, :1].permute(0, 3, 1, 2)
    assert float((got_row - ref_row).abs().max() / ref_row.abs().max()) <= 1e-3
    del outs
    dy1 = torch.randn(N, H, W, C, generator=g).to(dev)
    dy2 = torch.randn(N, H, W, C, generator=g).to(dev)
    d = ops.conv_desc([Source(x1)], N, H, W, C, (3, 3), 1, 1.0, ops.MATH_TF32)
    dws = []
    for dy in (dy1, dy2, dy1 + dy2):
        dw = torch.zeros(C, C, 3, 3, device=dev)
        ops.conv_wgrad(d, dy, dw)
        dws.append(dw)
    err = (dws[0] + dws[1] - dws[2]).abs().max() / dws[2].abs().max()
    assert float(err) <= 2e-3, float(err)
