"""wgrad_tc on every tensor-core layer shape of the bench workload's default Unet (the layer table of
tools/bench_layers.py: channels, kernel size, pooled and two-source inputs at the bench resolution;
batch 4 instead of 32 to keep the float64 reference small).  These shapes cover each plan the
bench runs: 3x3 layers as one CTA per kernel column sharing a staged x halo, 1x1 layers, and the
transposed orientation dW^T[ci][co] of the layers with few output channels (c5.0, c6.0, u2, u3).

dW against float64, per element, in tf32 and tf32x3 (the weight-gradient contraction of the
`tf32x3-full` mode), within the arithmetic model of tests/test_conv_exact_gpu.py:
    |dW - dW64| <= c(K) (sum_p |dy| |x|),  c = 2^-10 + (K+2) 2^-23 (tf32), 2^-18 + (K+2) 2^-23 (tf32x3)
with K = N H W; two launches bitwise equal; tf32x3 at least 2x more accurate than tf32 (norm-wise).
The exact suite asks 8x at K of a few thousand.  Here K reaches 10^6 (c6.0), where each pixel
range accumulates about 190 tiles (12,000 pixels) in fp32 in both modes, and that common error
narrows the gap (3.5x measured on c6.0).
"""
import pytest
import torch
import torch.nn.functional as F

from atomai_b200 import ops
from atomai_b200.ops import Source
from tools.bench_layers import LAYERS

BATCH = 4


def _c_mode(math, K):
    return (2.0 ** -10 if math == ops.MATH_TF32 else 2.0 ** -18) + (K + 2) * 2.0 ** -23


@pytest.mark.gpu
@pytest.mark.parametrize("name,H,cins,cout,ks,pool", LAYERS, ids=[l[0] for l in LAYERS])
def test_wgrad_bench_layer(cuda, name, H, cins, cout, ks, pool):
    dev = cuda
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    srcs, refs = [], []
    for ci in cins:
        s = 2 * H if pool else H
        x = torch.randn(BATCH, s, s, ci, device=dev, generator=g)
        sc = torch.rand(ci, device=dev, generator=g) + 0.5
        sh = torch.randn(ci, device=dev, generator=g) * 0.3
        srcs.append(Source(x, sc, sh, pool))
        # the loader's arithmetic: fmaf(x, scale, shift) rounded to fp32, then the 2x2 max
        xr = (x.double() * sc.double() + sh.double()).float().permute(0, 3, 1, 2).double()
        refs.append(F.max_pool2d(xr, 2, 2) if pool else xr)
    x64 = torch.cat(refs, 1)
    cin = x64.shape[1]
    dy = torch.randn(BATCH, H, H, cout, device=dev, generator=g)
    dy64 = dy.permute(0, 3, 1, 2).double()
    pad = ks // 2

    def wgrad64(x, d):
        w = torch.zeros(cout, cin, ks, ks, device=dev, dtype=torch.float64, requires_grad=True)
        F.conv2d(x, w, None, padding=pad).backward(d)
        return w.grad

    ref, m = wgrad64(x64, dy64), wgrad64(x64.abs(), dy64.abs())
    K = BATCH * H * H
    errs = {}
    for math in (ops.MATH_TF32, ops.MATH_TF32X3):
        d = ops.conv_desc(srcs, BATCH, H, H, cout, (ks, ks), 1, 1.0, math)
        assert ops.conv_supported(d, 1)
        runs = []
        for _ in range(2):
            dw = torch.zeros(cout, cin, ks, ks, device=dev)
            ops.conv_wgrad(d, dy, dw)
            runs.append(dw)
        torch.cuda.synchronize()
        err = (runs[0].double() - ref).abs()
        ratio = float((err / (_c_mode(math, K) * m).clamp_min(1e-300)).max())
        assert ratio <= 1.0, f"{name} math={math}: worst |dW - dW64| / bound = {ratio:.3g}"
        assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), \
            f"{name} math={math}: two launches differ"
        errs[math] = float(err.norm())
    assert errs[ops.MATH_TF32X3] <= errs[ops.MATH_TF32] / 2, \
        f"{name}: tf32x3 error {errs[ops.MATH_TF32X3]:.3g} not 2x below tf32 {errs[ops.MATH_TF32]:.3g}"
