"""Thin layers that take two tiles per consumer pass (conv_tc, ConvTcParams::pair = 2): the same
float64 parity as tests/test_conv_exact_gpu.py at the seams of the pairing (a lone last tile
per pipeline, a single pair per launch, ragged image edges, every k-chunk count), and bitwise equality
of outputs and BatchNorm statistics with one tile per pass (ATOMAI_B200_PAIR=0) on normal data."""
import ctypes as C
import os
import tempfile

import pytest
import torch

from atomai_b200 import _C, ops
from atomai_b200.ops import Source
from test_conv_exact_gpu import TF32, TF32X3, L, S, run_dgrad, run_fwd
from test_conv_plan_thin import TILE_RE

MATHS = [TF32, TF32X3]
MATH_IDS = ["tf32", "tf32x3"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pair_of(layer, math):
    """Tiles per consumer pass the plan gives `layer` (from the ATOMAI_B200_PLAN_LOG lines)."""
    from test_conv_plan import layer_desc
    old = os.environ.get("ATOMAI_B200_PLAN_LOG")
    os.environ["ATOMAI_B200_PLAN_LOG"] = "1"
    saved = os.dup(2)
    try:
        with tempfile.TemporaryFile() as f:
            os.dup2(f.fileno(), 2)
            try:
                g, b, s = C.c_int(), C.c_int(), C.c_int()
                _C.lib().atomai_b200_conv_info(C.byref(layer_desc(layer, math)), C.byref(g), C.byref(b),
                                               C.byref(s))
            finally:
                os.dup2(saved, 2)
            f.seek(0)
            text = f.read().decode(errors="replace")
    finally:
        os.close(saved)
        if old is None:
            del os.environ["ATOMAI_B200_PLAN_LOG"]
        else:
            os.environ["ATOMAI_B200_PLAN_LOG"] = old
    m = TILE_RE.search(text)
    assert m, text
    return int(m.group(2))


def seam_layers():
    sms = _sms()
    return [
        # tiles = 4 * SMs + k: pipeline 0 of the first k CTAs ends on a lone tile (k = 1, 2), or
        # pipeline 1 does (k = -1, 3); 1 and 3 k-chunks per tile
        ("4sms", L([16], 32, 8, 8 * 4 * sms, N=1)),
        ("4sms+1", L([48], 16, 8, 8 * (4 * sms + 1), N=1)),
        ("4sms+2", L([16], 32, 8, 8 * (4 * sms + 2), N=1)),
        ("4sms+3", L([16], 32, 8, 8 * (4 * sms + 3), N=1)),
        ("4sms-1", L([48], 16, 8, 8 * (4 * sms - 1), N=1)),
        # 2 * SMs + 1 tiles: only pipeline 0 of the first CTA has a pair, every other pass is a
        # lone tile
        ("2sms+1", L([16], 16, 8, 8 * (2 * sms + 1), N=1)),
        # ragged edges of several images, two sources, pooled source
        # (enough images for more than two tiles per CTA)
        ("ragged_cat", L([8, 8], 16, 13, 21, N=64)),
        ("ragged_pool", L([S(16, ops.SRC_POOL, aff=True)], 32, 11, 19, N=64)),
        ("affine_k8", L([S(8, aff=True)], 16, 16, 24, N=64)),
    ]


SEAM_IDS = ["4sms", "4sms+1", "4sms+2", "4sms+3", "4sms-1", "2sms+1", "ragged_cat", "ragged_pool",
            "affine_k8"]


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("idx", range(len(SEAM_IDS)), ids=SEAM_IDS)
def test_paired_forward_exact(cuda, idx, math):
    tag, layer = seam_layers()[idx]
    assert pair_of(layer, math) == 2, tag
    run_fwd(layer, math, cuda, tag=tag, amp=1, stats=all(s.tr == ops.SRC_PLAIN and not s.aff
                                                          for s in layer.srcs))
    run_fwd(layer, math, cuda, tag=tag + "/slope0.25", amp=1, slope=0.25, out="slice", seed=1)


@pytest.mark.gpu
def test_few_tiles_stay_unpaired(cuda):
    """With at most two tiles per CTA every pass would be a lone tile: the plan keeps one tile per
    pass there."""
    sms = _sms()
    for layer in (L([16], 16, 8, 8 * (sms - 1), N=1), L([16], 32, 8, 8 * 2 * sms, N=1)):
        assert pair_of(layer, TF32X3) == 1, layer
    assert pair_of(L([16], 32, 8, 8 * (2 * sms + 1), N=1), TF32X3) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("tag,layer", [("d16_32", L([32], 16, 16, 40, N=32)),
                                       ("d_cat_16_16", L([16, 16], 16, 13, 21, N=64)),
                                       ("d32_16", L([32], 16, 8, 8 * 67, N=4))],
                         ids=["d16_32", "d_cat_16_16", "d32_16"])
def test_paired_dgrad_exact(cuda, tag, layer, math):
    # the data gradient is a forward convolution of dy (cout channels) onto ctot channels
    assert pair_of(L([layer.cout], layer.ctot, layer.H, layer.W, N=layer.N), math) == 2, tag
    run_dgrad(layer, math, cuda, tag=tag, amp=1)


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS, ids=MATH_IDS)
@pytest.mark.parametrize("shape", [(32, [16, 16], 16, 64), (4, [48], 32, 96), (12, [16], 16, 37)],
                         ids=["c6_like", "c5_like", "ragged"])
def test_pairing_bitwise_equal_to_single_tiles(cuda, monkeypatch, math, shape):
    """Normal data: the paired and the one-tile-per-pass kernel give identical bits, outputs and
    statistics (each tile keeps its MMA order and its place in the statistics order)."""
    n, cins, cout, hw = shape
    g = torch.Generator().manual_seed(7)
    srcs = []
    for ci in cins:
        x = torch.randn(n, hw, hw, ci, generator=g).to(cuda)
        srcs.append(Source(x, (torch.rand(ci, generator=g) + 0.5).to(cuda),
                           torch.randn(ci, generator=g).to(cuda)))
    w = (torch.randn(cout, sum(cins), 3, 3, generator=g) * 0.1).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda)
    d = ops.conv_desc(srcs, n, hw, hw, cout, (3, 3), 1, 0.01, math)
    wp = ops.prep_weights(w, ops.WMODE_FWD, math)
    outs = []
    for pair in ("1", "0"):
        monkeypatch.setenv("ATOMAI_B200_PAIR", pair)
        y = torch.full((n, hw, hw, cout), float("nan"), device=cuda)
        st = torch.zeros(2 * cout, device=cuda, dtype=torch.float64)
        ops.conv_fwd(d, wp, b, y, st)
        torch.cuda.synchronize()
        outs.append((y, st))
    monkeypatch.setenv("ATOMAI_B200_PAIR", "1")
    layer = L(cins, cout, hw, hw, N=n)
    assert pair_of(layer, math) == 2
    (y1, s1), (y0, s0) = outs
    assert not torch.isnan(y1).any()
    assert torch.equal(y1.view(torch.int32), y0.view(torch.int32))
    assert torch.equal(s1.view(torch.int64), s0.view(torch.int64))
