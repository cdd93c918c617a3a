"""
MobileNetV2 layers on the native tape (atomai_b200/engine.py): the Regressor / Classifier backbone
(atomai/nets/blocks.py:376-387, torchvision's mobilenet_v2 feature extractor).

MobileNetV2 orders a layer conv -> BatchNorm -> ReLU6, so an activation carries the pending
transform relu6(scale * t + shift) (`Relu6Act`) instead of the engine's plain affine.  Consumers:
  * the depthwise 3x3 convolution and the pooled head apply it while loading (mobilenet.cu);
  * the 1x1 projection after a depthwise layer runs on conv_tc, which applies an affine only, so
    the activation is written out first (`materialize_relu6`).
Backward recomputes the ReLU6 mask 0 < scale * t + shift < 6 from the stored raw t.

The 1x1 layers (expand, project, 320 -> 1280) go to conv_tc / wgrad_tc whenever
`ops.tc_supported` takes them, and to the exact-fp32 kernels otherwise (Cout = 24, or math mode
'fp32'), exactly as `Tape.conv` chooses.  conv_tc takes at most 256 output channels, so wider layers
run as column blocks writing channel slices of one buffer (as `Tape.mlp` does), and their data
gradients as blocks of input channels.  A 1x1 convolution does not depend on the pixel layout, so
its tensors are presented as one (1, P/8, 8, C) image: the 2x2 and 1x1 maps of small inputs then
fill the tiles as well as large ones do.

BatchNorm statistics, BatchNorm-backward sums and weight gradients are ordered sums, and go through
the tape's `comm` hooks under data parallelism like those of `Tape.conv`.
"""
from typing import List, Optional, Tuple

import torch

from . import engine, ops
from .engine import Act, Tape, _acc_grad, _d
from .ops import ACT_LRELU, MATH_FP32, Source

_MAX_COUT = 256        # widest output block of conv_tc


class Relu6Act(Act):
    """Activation whose pending transform is relu6(scale * t + shift).  Only the MobileNet layers
    of this module read it; it has no conv-engine `Source`.  `pool_grad`: the (N, 1, 1, C)
    gradient of an average pool of this activation, not yet spread over the pixels: the
    producer's BatchNorm backward reads it broadcast when it is the only gradient."""
    __slots__ = ("pool_grad",)

    def __init__(self, *args, **kwargs):
        super(Relu6Act, self).__init__(*args, **kwargs)
        self.pool_grad = None

    def source(self) -> Source:
        raise RuntimeError("a pending ReLU6 is applied by the MobileNet kernels or materialised "
                           "with materialize_relu6, not by the convolution engine")


def _blocks(c: int) -> List[Tuple[int, int]]:
    """Column blocks of <= 256 channels, multiples of 16 where the width allows."""
    if c <= _MAX_COUT:
        return [(0, c)]
    nblk = -(-c // _MAX_COUT)
    per = -(-(c // 16) // nblk) * 16
    return [(c0, min(c, c0 + per)) for c0 in range(0, c, per)]


def _flat(t: torch.Tensor) -> torch.Tensor:
    """(N, H, W, C[ld]) -> (1, P/8, 8, C[ld]) view when the pixels allow it (1x1 layers only)."""
    n, h, w, c = t.shape
    p = n * h * w
    if p % 8:
        return t
    ld = ops._ld(t)
    return t.as_strided((1, p // 8, 8, c), (p * ld, 8 * ld, ld, 1))


def _bn_forward(tape: Tape, bn, stats: Optional[torch.Tensor], blocks, count: int, dev):
    """BatchNorm of a layer whose raw output sums of block (c0, c1) are stats[2*c0 : 2*c1]
    (sum y, then sum y^2).  Returns (scale, shift, mean, invstd, count)."""
    cout = bn.num_features
    scale = torch.empty(cout, device=dev, dtype=torch.float32)
    shift = torch.empty(cout, device=dev, dtype=torch.float32)
    if stats is None:
        ops.bn_finalize(None, count, _d(bn.weight), _d(bn.bias), bn.running_mean, bn.running_var,
                        0.0, bn.eps, False, scale, shift, None, None)
        return scale, shift, None, None, count
    mean = torch.empty(cout, device=dev, dtype=torch.float32)
    invstd = torch.empty(cout, device=dev, dtype=torch.float32)
    mom = bn.momentum if bn.momentum is not None else 0.1
    if tape.comm is not None:
        count = tape.comm.allreduce_count(count)
        tape.comm.allreduce_sum_(stats)
    sl = lambda t, c0, c1: None if t is None else t[c0:c1]   # noqa: E731
    for c0, c1 in blocks:
        ops.bn_finalize(stats[2 * c0:2 * c1], count, sl(_d(bn.weight), c0, c1),
                        sl(_d(bn.bias), c0, c1), sl(bn.running_mean, c0, c1),
                        sl(bn.running_var, c0, c1), mom, bn.eps, True, scale[c0:c1],
                        shift[c0:c1], mean[c0:c1], invstd[c0:c1])
    if bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
    return scale, shift, mean, invstd, count


def _bn_backward(tape: Tape, rec, dy: torch.Tensor) -> torch.Tensor:
    """Gradient before the BatchNorm (and ReLU6) of `rec.out` from the gradient after them."""
    out, bn = rec.out, rec.bn
    a = out.t
    cout = a.shape[3]
    dev = a.device
    sums = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
    if isinstance(out, Relu6Act):
        g = torch.empty(a.shape, device=dev, dtype=torch.float32)
        ops.relu6_bwd_reduce(dy, a, out.scale, out.shift, rec.mean, rec.invstd, g, sums,
                             pooled=dy.shape[1:3] != a.shape[1:3])
        dy = g
    else:
        ops.bn_bwd_reduce(dy, a, rec.mean, rec.invstd, sums)
    tape._add_pgrad(bn.bias, sums[:cout].float())
    tape._add_pgrad(bn.weight, sums[cout:].float())
    if tape.comm is not None:
        tape.comm.allreduce_sum_(sums)
    dpre = torch.empty(a.shape, device=dev, dtype=torch.float32)
    # bn_lrelu_bwd takes up to 1024 channels: the 1280-wide layer goes in channel blocks
    for c0, c1 in _blocks(cout):
        sl = slice(c0, c1)
        bsums = sums if (c0, c1) == (0, cout) else torch.cat((sums[sl], sums[cout + c0:cout + c1]))
        ops.bn_act_bwd(dy[..., sl], a[..., sl], rec.mean[sl], rec.invstd[sl], out.scale[sl], bsums,
                       rec.count, None, ACT_LRELU, 1.0, dpre[..., sl], None)
    return dpre


def _take_grad(out: Act) -> Optional[torch.Tensor]:
    """The gradient w.r.t. `out`: its pooled (N, 1, 1, C) gradient when that is all there is
    (read broadcast by relu6_bwd_reduce), else the full-resolution sum of all contributions."""
    dy, pg = out.grad, getattr(out, "pool_grad", None)
    out.grad = None
    if pg is None:
        return dy
    out.pool_grad = None
    if dy is None:
        return pg
    g = torch.empty(out.t.shape, device=pg.device, dtype=torch.float32)
    ops.avgpool_bwd(pg, g)
    ops.add_slice(dy, g, True)
    return g


def _use_batch_stats(tape: Tape, bn) -> bool:
    return tape.training or bn.running_mean is None


class _LayerRec:
    __slots__ = ("x", "out", "conv", "bn", "mean", "invstd", "count", "blocks", "math", "stride",
                 "depthwise")

    def _check_training(self):
        assert self.mean is not None, "backward through eval-mode BatchNorm is not supported"


class _PwRec(_LayerRec):
    """1x1 convolution (no bias) -> BatchNorm [-> ReLU6] on conv_tc / wgrad_tc."""

    def backward(self, tape: Tape) -> None:
        out, x = self.out, self.x
        dy = _take_grad(out)
        if dy is None:
            return
        self._check_training()
        dpre = _bn_backward(tape, self, dy)
        wt = self.conv.weight
        cout, cin = wt.shape[0], wt.shape[1]
        dev = dpre.device
        xs = Source(_flat(x.t), x.scale, x.shift)
        dflat = _flat(dpre)
        _, fh, fw, _ = dflat.shape
        fn = dflat.shape[0]
        dw = torch.zeros((cout, cin, 1, 1), device=dev, dtype=torch.float32)
        for (c0, c1), math in zip(self.blocks, self.math):
            wmath = math if (math == MATH_FP32 or engine._MATH["wgrad"] is None) \
                else engine._MATH["wgrad"]
            dsc = ops.conv_desc([xs], fn, fh, fw, c1 - c0, (1, 1), 1, 1.0, wmath)
            if wmath != MATH_FP32 and not (engine._MATH["wgrad_tc"] and ops.conv_supported(dsc, 1)):
                dsc.math = MATH_FP32
            ops.conv_wgrad(dsc, dflat[..., c0:c1], dw[c0:c1])
        tape._add_pgrad(wt, dw)
        if not x.needs_grad:
            return
        dx = torch.empty(x.t.shape, device=dev, dtype=torch.float32)
        dxf = _flat(dx)
        w = wt.detach()
        for k0, k1 in _blocks(cin):
            dsrc = [Source(dflat)]
            dmath = engine._MATH["mode"] if (engine._MATH["mode"] != MATH_FP32 and
                                             ops.tc_supported(dsrc, k1 - k0)) else MATH_FP32
            wpd = ops.prep_weights(w[:, k0:k1].contiguous(), ops.WMODE_DGRAD, dmath)
            dd = ops.conv_desc(dsrc, fn, fh, fw, k1 - k0, (1, 1), 1, 1.0, dmath)
            ops.conv_fwd(dd, wpd, None, dxf[..., k0:k1], None)
        _acc_grad(x, dx, True)


def pointwise(tape: Tape, x: Act, conv, bn, relu6: bool) -> Act:
    """conv (1x1, no bias) -> BatchNorm [-> ReLU6]; x: plain or pending-affine activation."""
    if isinstance(x, Relu6Act):
        x = materialize_relu6(tape, x)
    n, h, w, cin = x.shape
    wt = conv.weight
    cout = wt.shape[0]
    assert wt.shape[1] == cin and wt.shape[2:] == (1, 1) and conv.bias is None
    dev = wt.device
    y = torch.empty((n, h, w, cout), device=dev, dtype=torch.float32)
    xs = Source(_flat(x.t), x.scale, x.shift)
    yf = _flat(y)
    fn, fh, fw, _ = yf.shape
    stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64) \
        if _use_batch_stats(tape, bn) else None
    blocks = _blocks(cout)
    maths = []
    for c0, c1 in blocks:
        math = engine._MATH["mode"] if (engine._MATH["mode"] != MATH_FP32 and
                                        ops.tc_supported([xs], c1 - c0)) else MATH_FP32
        d = ops.conv_desc([xs], fn, fh, fw, c1 - c0, (1, 1), 1, 1.0, math)
        wp = ops.prep_weights(wt.detach()[c0:c1], ops.WMODE_FWD, math)
        ops.conv_fwd(d, wp, None, yf[..., c0:c1], None if stats is None else stats[2 * c0:2 * c1])
        maths.append(math)
    tape.widths.append(w)
    scale, shift, mean, invstd, count = _bn_forward(tape, bn, stats, blocks, n * h * w, dev)
    out = (Relu6Act if relu6 else Act)(y, scale, shift)
    if tape.record:
        r = _PwRec()
        r.x, r.out, r.conv, r.bn, r.mean, r.invstd, r.count = x, out, conv, bn, mean, invstd, count
        r.blocks, r.math = blocks, maths
        tape.ops.append(("custom", r))
    return out


class _Conv3Rec(_LayerRec):
    """3x3 convolution (stem or depthwise) -> BatchNorm -> ReLU6 on the mobilenet.cu kernels."""

    def backward(self, tape: Tape) -> None:
        out, x = self.out, self.x
        dy = _take_grad(out)
        if dy is None:
            return
        self._check_training()
        dpre = _bn_backward(tape, self, dy)
        clip = isinstance(x, Relu6Act)
        dw = torch.zeros(self.conv.weight.shape, device=dpre.device, dtype=torch.float32)
        ops.conv3x3_wgrad(dpre, x.t, x.scale, x.shift, clip, self.depthwise, dw, self.stride)
        tape._add_pgrad(self.conv.weight, dw)
        if x.needs_grad:
            dx = torch.empty(x.t.shape, device=dpre.device, dtype=torch.float32)
            ops.dw3x3_dgrad(dpre, self.conv.weight.detach().contiguous(), dx, self.stride)
            _acc_grad(x, dx, True)


def conv3x3(tape: Tape, x: Act, conv, bn) -> Relu6Act:
    """Conv2d(3x3, pad 1, stride 1|2, groups 1 or C, no bias) -> BatchNorm -> ReLU6.  x: a plain,
    pending-affine or pending-ReLU6 activation."""
    n, h, w, cin = x.shape
    wt = conv.weight
    cout = wt.shape[0]
    stride = conv.stride[0]
    depthwise = conv.groups > 1
    assert wt.shape[2:] == (3, 3) and conv.padding == (1, 1) and conv.stride[0] == conv.stride[1] \
        and conv.bias is None and conv.dilation == (1, 1)
    assert (depthwise and conv.groups == cin == cout) or (not depthwise and wt.shape[1] == cin)
    if x.needs_grad and not depthwise and tape.record:
        raise NotImplementedError("the data gradient of the dense 3x3 stem is not implemented")
    dev = wt.device
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    y = torch.empty((n, ho, wo, cout), device=dev, dtype=torch.float32)
    stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64) \
        if _use_batch_stats(tape, bn) else None
    ops.conv3x3_fwd(x.t, x.scale, x.shift, isinstance(x, Relu6Act), wt.detach().contiguous(),
                    depthwise, y, stride, stats)
    tape.widths.append(wo)
    blocks = [(0, cout)]
    scale, shift, mean, invstd, count = _bn_forward(tape, bn, stats, blocks, n * ho * wo, dev)
    out = Relu6Act(y, scale, shift)
    if tape.record:
        r = _Conv3Rec()
        r.x, r.out, r.conv, r.bn, r.mean, r.invstd, r.count = x, out, conv, bn, mean, invstd, count
        r.stride, r.depthwise = stride, depthwise
        tape.ops.append(("custom", r))
    return out


class _MatRelu6Rec:
    def __init__(self, x, out):
        self.x, self.out = x, out

    def backward(self, tape: Tape) -> None:
        g = self.out.grad
        self.out.grad = None
        if g is not None and self.x.needs_grad:
            _acc_grad(self.x, g, self.out.grad_owned)


def materialize_relu6(tape: Tape, x: Relu6Act) -> Act:
    """relu6(scale * t + shift) written out (gradient passes through; the mask is applied by the
    producer's backward)."""
    y = torch.empty(x.t.shape, device=x.t.device, dtype=torch.float32)
    ops.affine_relu6(x.t, x.scale, x.shift, y)
    out = Act(y, needs_grad=x.needs_grad)
    if tape.record:
        tape.ops.append(("custom", _MatRelu6Rec(x, out)))
    return out


class _PoolRec:
    def __init__(self, x, out):
        self.x, self.out = x, out

    def backward(self, tape: Tape) -> None:
        dy = self.out.grad
        self.out.grad = None
        if dy is None or not self.x.needs_grad:
            return
        # kept per image: the producer's BatchNorm backward spreads it over the pixels while
        # reducing, so no (N, H, W, C) gradient is written (_take_grad)
        if self.x.pool_grad is None:
            self.x.pool_grad = engine._dense(dy)
        else:
            acc = engine._dense(self.x.pool_grad).clone()
            ops.add_slice(dy, acc, True)
            self.x.pool_grad = acc


def avgpool(tape: Tape, x: Relu6Act) -> Act:
    """AdaptiveAvgPool2d(1) + flatten of relu6(scale * t + shift): (N, 1, 1, C)."""
    n, _, _, c = x.t.shape
    y = torch.empty((n, 1, 1, c), device=x.t.device, dtype=torch.float32)
    ops.avgpool_relu6_fwd(x.t, x.scale, x.shift, y)
    out = Act(y, needs_grad=x.needs_grad)
    if tape.record:
        tape.ops.append(("custom", _PoolRec(x, out)))
    return out


def linear(tape: Tape, x: Act, lin) -> Act:
    """nn.Linear on the (B, 1, 1, K) pooled features.  Forward on the `gemm` kernel (fixed
    summation order, so training stays bit-reproducible), backward through the tape's Linear
    backward (`linear_bwd`)."""
    b, k = x.t.shape[0], x.t.shape[3]
    assert x.t.shape[1:3] == (1, 1) and x.t.is_contiguous() and not x.pending()
    w = lin.weight.detach()
    o = w.shape[0]
    y = torch.empty((b, 1, 1, o), device=w.device, dtype=torch.float32)
    ops.gemm(x.t, k, 1, w, 1, k, y, o, b, o, k, _d(lin.bias), ACT_LRELU, 1.0)
    out = Act(y, needs_grad=True)
    if tape.record:
        tape.ops.append(("lin", (x, out, lin, None)))
    return out


class _LogSoftmaxRec:
    def __init__(self, x, out):
        self.x, self.out = x, out

    def backward(self, tape: Tape) -> None:
        dy = self.out.grad
        self.out.grad = None
        if dy is None or not self.x.needs_grad:
            return
        b, c = self.out.t.shape[0], self.out.t.shape[3]
        dx = torch.empty_like(self.out.t)
        ops.log_softmax_bwd(self.out.t.view(b, c), engine._dense(dy).view(b, c), dx.view(b, c))
        _acc_grad(self.x, dx, True)


def log_softmax(tape: Tape, x: Act) -> Act:
    """LogSoftmax(dim=1) of a (B, 1, 1, C) activation."""
    b, c = x.t.shape[0], x.t.shape[3]
    y = torch.empty((b, 1, 1, c), device=x.t.device, dtype=torch.float32)
    ops.log_softmax_fwd(x.t.reshape(b, c), y.view(b, c))
    out = Act(y, needs_grad=x.needs_grad)
    if tape.record:
        tape.ops.append(("custom", _LogSoftmaxRec(x, out)))
    return out
