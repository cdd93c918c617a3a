"""
Thin tensor-level wrappers over the C ABI (include/atomai_b200.h).

torch is used here for device memory and the current stream only; every
function launches hand-written sm_90a kernels from libatomai_b200.so and
raises if that library is unavailable.  Activations are NHWC fp32 tensors of
shape (N, H, W, C); a channel slice of a wider tensor is passed as a view whose
last-dim stride is 1 (its pixel stride `ld` is read from the strides).
"""
import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _C
from ._C import (ACT_LRELU, ACT_TANH, MATH_FP32, MATH_TF32, MATH_TF32X3, WMODE_DGRAD, WMODE_FWD, check,
                 lib, ptr, stream_ptr)


def _ld(t: torch.Tensor) -> int:
    """Pixel stride of an NHWC (view) tensor; validates the layout (size-1 dims are free)."""
    assert t.dtype == torch.float32 and t.is_cuda, "fp32 CUDA tensor expected"
    assert t.dim() == 4, f"NHWC tensor expected, got shape {tuple(t.shape)}"
    if t.is_contiguous():
        return t.shape[3]
    N, H, W, Cc = t.shape
    st = t.stride()
    assert Cc == 1 or st[3] == 1, f"channels must be innermost, strides {st}"
    ld = st[2] if W > 1 else (st[1] if H > 1 else (st[0] if N > 1 else Cc))
    assert ld >= Cc and (W == 1 or st[2] == ld) and (H == 1 or st[1] == ld * W) and \
        (N == 1 or st[0] == ld * W * H), \
        f"pixel-major layout expected, got shape {tuple(t.shape)} strides {st}"
    return ld


SRC_PLAIN, SRC_POOL, SRC_UP_BILINEAR, SRC_UP_NEAREST = 0, 1, 2, 3


class Source:
    """One conv input: NHWC tensor + optional pending BN affine + optional on-load resampling
    (`pool`: False/0 none, True/1 2x2 max-pool of a (2H, 2W) tensor, 2 / 3 bilinear / nearest 2x
    upsampling of a (H/2, W/2) tensor)."""
    __slots__ = ("t", "scale", "shift", "pool")

    def __init__(self, t, scale=None, shift=None, pool=False):
        self.t, self.scale, self.shift, self.pool = t, scale, shift, int(pool)

    @property
    def C(self):
        return self.t.shape[3]


def conv_desc(srcs: Sequence[Source], N, H, W, Cout, ks=(3, 3), dil=1, lrelu=1.0,
              math=MATH_TF32, out_nchw=False, act=ACT_LRELU) -> _C.Conv:
    d = _C.Conv()
    d.N, d.H, d.W, d.Cout = N, H, W, Cout
    d.ks_h, d.ks_w, d.dil = ks[0], ks[1], dil
    d.nsrc = len(srcs)
    for i, s in enumerate(srcs):
        e = d.src[i]
        e.ptr = s.t.data_ptr()
        e.scale = ptr(s.scale)
        e.shift = ptr(s.shift)
        e.C = s.t.shape[3]
        e.ld = _ld(s.t)
        e.pool = int(s.pool)
        sh, sw = s.t.shape[1], s.t.shape[2]
        if s.pool == SRC_POOL:
            assert (sh, sw) == (2 * H, 2 * W), f"pooled source must be {(2*H, 2*W)}, got {(sh, sw)}"
        elif s.pool in (SRC_UP_BILINEAR, SRC_UP_NEAREST):
            assert (2 * sh, 2 * sw) == (H, W), f"upsampled source must be {(H//2, W//2)}, got {(sh, sw)}"
        else:
            assert (sh, sw) == (H, W), f"source spatial {(sh, sw)} != {(H, W)}"
        assert s.t.shape[0] == N
    d.lrelu = float(lrelu)
    d.math = math
    d.out_nchw = 1 if out_nchw else 0
    d.act = act
    return d


def tc_supported(srcs: Sequence[Source], Cout: int) -> bool:
    """Shapes the wgmma conv path takes (mirrors ab_conv_tc_supported)."""
    ctot = sum(s.C for s in srcs)
    return (all(s.C % 4 == 0 and _ld(s.t) % 4 == 0 and s.t.data_ptr() % 16 == 0 for s in srcs)
            and ctot % 8 == 0 and Cout % 16 == 0 and 16 <= Cout <= 256)


def conv_supported(d: _C.Conv, which: int = 0) -> bool:
    """Does the wgmma kernel take this descriptor?  which: 0 forward/dgrad, 1 weight gradient
    (atomai_b200_conv_supported — the single source of truth, no Python mirror)."""
    return bool(lib().atomai_b200_conv_supported(C.byref(d), which))


def prep_weights(w_oihw: torch.Tensor, mode: int, math: int) -> torch.Tensor:
    """OIHW (or OIW for 1-D) conv weight -> kernel layout for `math` / `mode`."""
    w = w_oihw.detach()
    if w.dim() == 3:
        w = w.unsqueeze(2)
    w = w.contiguous()
    Cout, Cin, kh, kw = w.shape
    n = lib().atomai_b200_prep_weights_elems(Cout, Cin, kh, kw, mode, math)
    out = torch.empty(n, device=w.device, dtype=torch.float32)
    check(lib().atomai_b200_prep_weights(ptr(w), Cout, Cin, kh, kw, mode, math, ptr(out),
                                         stream_ptr()))
    return out


# Optional per-launch timing of the convolution family (bench.py's live roofline): a list that
# receives (kernel, algorithmic FLOPs, algorithmic bytes, start event, end event) per launch.
PROFILE = None


def _conv_work(d: _C.Conv):
    ctot = sum(d.src[i].C for i in range(d.nsrc))
    pix = d.N * d.H * d.W
    flops = 2.0 * pix * d.ks_h * d.ks_w * ctot * d.Cout
    rd = sum(d.src[i].C * (4 if d.src[i].pool else 1) for i in range(d.nsrc))
    return flops, 4.0 * pix * (rd + d.Cout)


def _timed(kernel: str, d: _C.Conv, fn) -> None:
    if PROFILE is None:
        fn()
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    fl, by = _conv_work(d)
    PROFILE.append((kernel, fl, by, e0, e1))


def conv_fwd(d: _C.Conv, w_prepped, bias, out: torch.Tensor, stats=None) -> None:
    ld_y = d.Cout if d.out_nchw else _ld(out)
    _timed("conv_tc_kernel" if d.math != MATH_FP32 else "conv_simt",  d, lambda: check(
        lib().atomai_b200_conv_fwd(C.byref(d), ptr(w_prepped), ptr(bias), ptr(out), ld_y,
                                   ptr(stats), stream_ptr())))


def conv_wgrad(d: _C.Conv, dy: torch.Tensor, dw_oihw: torch.Tensor) -> None:
    _timed("wgrad_tc_kernel" if d.math != MATH_FP32 else "wgrad_simt", d, lambda: check(
        lib().atomai_b200_conv_wgrad(C.byref(d), ptr(dy), _ld(dy), ptr(dw_oihw), stream_ptr())))


def bn_finalize(stats, count, gamma, beta, rmean, rvar, momentum, eps, training, scale, shift,
                mean=None, invstd=None) -> None:
    check(lib().atomai_b200_bn_finalize(ptr(stats), scale.numel(), float(count), ptr(gamma),
                                        ptr(beta), ptr(rmean), ptr(rvar), momentum, eps,
                                        1 if training else 0, ptr(scale), ptr(shift), ptr(mean),
                                        ptr(invstd), stream_ptr()))


def affine(a: torch.Tensor, scale, shift, out: torch.Tensor, out_nchw=False) -> None:
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_affine(ptr(a), _ld(a), ptr(scale), ptr(shift), ptr(out),
                                   Cc if out_nchw else _ld(out), N * H * W, Cc,
                                   H * W if out_nchw else 0, stream_ptr()))


def bn_bwd_reduce(dy, a, mean, invstd, sums) -> None:
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_bn_bwd_reduce(ptr(dy), _ld(dy), ptr(a), _ld(a), ptr(mean),
                                          ptr(invstd), N * H * W, Cc, ptr(sums), stream_ptr()))


def bn_act_bwd(dy, a, mean, invstd, scale, sums, count, extra, act, slope, dpre, dbias) -> None:
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_bn_lrelu_bwd(
        ptr(dy), _ld(dy) if dy is not None else 0, ptr(a), _ld(a), ptr(mean), ptr(invstd),
        ptr(scale), ptr(sums), float(count), ptr(extra), _ld(extra) if extra is not None else 0,
        act, float(slope), ptr(dpre), _ld(dpre), ptr(dbias), N * H * W, Cc, stream_ptr()))


def pool_fwd(a, scale, shift, out) -> None:
    N, Ho, Wo, Cc = out.shape
    check(lib().atomai_b200_pool2x2_fwd(ptr(a), _ld(a), ptr(scale), ptr(shift), ptr(out),
                                        _ld(out), N, Ho, Wo, Cc, stream_ptr()))


def pool_bwd(dp, a, scale, shift, dfull, accumulate, mean=None, invstd=None, sums=None) -> None:
    """dfull (+)= unpool(dp); with `sums` also the BatchNorm-backward reductions of the result."""
    N, Ho, Wo, Cc = dp.shape
    check(lib().atomai_b200_pool2x2_bwd_bn(ptr(dp), _ld(dp), ptr(a), _ld(a), ptr(scale), ptr(shift),
                                           ptr(dfull), _ld(dfull), 1 if accumulate else 0, N, Ho, Wo,
                                           Cc, ptr(mean), ptr(invstd), ptr(sums), stream_ptr()))


def pool_bwd_stats_ok(C: int) -> bool:
    c4 = C // 4
    return C % 4 == 0 and c4 >= 1 and (c4 & (c4 - 1)) == 0 and c4 <= 256


def upsample_fwd(x, out, bilinear=True) -> None:
    N, h, w, Cc = x.shape
    check(lib().atomai_b200_upsample2x_fwd(ptr(x), _ld(x), ptr(out), _ld(out), N, h, w, Cc,
                                           1 if bilinear else 0, stream_ptr()))


def upsample_bwd(dy, dx, bilinear=True) -> None:
    N, h, w, Cc = dx.shape
    check(lib().atomai_b200_upsample2x_bwd(ptr(dy), _ld(dy), ptr(dx), _ld(dx), N, h, w, Cc,
                                           1 if bilinear else 0, stream_ptr()))


def avgpool_fwd(x, out, sh: int, sw: int) -> None:
    """out (N, H//sh, W//sw, C) = sh x sw window averages of x (N, H, W, C)."""
    N, H, W, Cc = x.shape
    check(lib().atomai_b200_avgpool_fwd(ptr(x), _ld(x), ptr(out), _ld(out), N, H, W, Cc, int(sh),
                                        int(sw), stream_ptr()))


def upsample_w2x_fwd(x, out) -> None:
    """Nearest x2 along the width of a (N, 1, w, C) signal."""
    N, _, w, Cc = x.shape
    check(lib().atomai_b200_upsample_w2x_fwd(ptr(x), _ld(x), ptr(out), _ld(out), N, w, Cc,
                                             stream_ptr()))


def upsample_w2x_bwd(dy, dx) -> None:
    N, _, w, Cc = dx.shape
    check(lib().atomai_b200_upsample_w2x_bwd(ptr(dy), _ld(dy), ptr(dx), _ld(dx), N, w, Cc,
                                             stream_ptr()))


def affine_res_act(a, scale, shift, res, slope, out) -> None:
    """out = LeakyReLU(a*scale + shift + res) (scale/shift/res optional)."""
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_affine_res_act(ptr(a), _ld(a), ptr(scale), ptr(shift), ptr(res),
                                           _ld(res) if res is not None else 0, float(slope),
                                           ptr(out), _ld(out), N * H * W, Cc, stream_ptr()))


def lrelu_mask_bwd(dy, y, slope, g) -> None:
    N, H, W, Cc = y.shape
    check(lib().atomai_b200_lrelu_mask_bwd(ptr(dy), _ld(dy), ptr(y), _ld(y), float(slope), ptr(g),
                                           _ld(g), N * H * W, Cc, stream_ptr()))


def resize_fwd(x, out, factor, bilinear=True) -> None:
    N, h, w, Cc = x.shape
    check(lib().atomai_b200_resize_fwd(ptr(x), _ld(x), ptr(out), _ld(out), N, h, w, Cc, int(factor),
                                       1 if bilinear else 0, stream_ptr()))


def resize_bwd(dy, dx, factor, bilinear=True) -> None:
    N, h, w, Cc = dx.shape
    check(lib().atomai_b200_resize_bwd(ptr(dy), _ld(dy), ptr(dx), _ld(dx), N, h, w, Cc, int(factor),
                                       1 if bilinear else 0, stream_ptr()))


def conv3x3_fwd(x, scale, shift, clip, w, depthwise, y, stride, stats=None) -> None:
    """y = conv3x3(act(x)), pad 1 (MobileNetV2 stem / depthwise), act = [relu6](x*scale + shift)."""
    N, H, W, Cin = x.shape
    Cout = y.shape[3]
    assert w.is_contiguous() and y.shape[1:3] == ((H - 1) // stride + 1, (W - 1) // stride + 1)
    check(lib().atomai_b200_conv3x3_fwd(ptr(x), _ld(x), ptr(scale), ptr(shift), 1 if clip else 0,
                                        ptr(w), 1 if depthwise else 0, ptr(y), _ld(y), N, H, W, Cin,
                                        Cout, stride, ptr(stats), stream_ptr()))


def conv3x3_wgrad(dy, x, scale, shift, clip, depthwise, dw, stride) -> None:
    """dw (OIHW, zeroed) += weight gradient of conv3x3_fwd."""
    N, H, W, Cin = x.shape
    assert dw.is_contiguous()
    check(lib().atomai_b200_conv3x3_wgrad(ptr(dy), _ld(dy), ptr(x), _ld(x), ptr(scale), ptr(shift),
                                          1 if clip else 0, 1 if depthwise else 0, ptr(dw), N, H, W,
                                          Cin, dy.shape[3], stride, stream_ptr()))


def dw3x3_dgrad(dy, w, dx, stride) -> None:
    """dx (N, H, W, C) = data gradient of the depthwise conv3x3_fwd w.r.t. its activated input."""
    N, H, W, Cc = dx.shape
    assert w.is_contiguous()
    check(lib().atomai_b200_dw3x3_dgrad(ptr(dy), _ld(dy), ptr(w), ptr(dx), _ld(dx), N, H, W, Cc,
                                        stride, stream_ptr()))


def relu6_bwd_reduce(dy, a, scale, shift, mean, invstd, g, sums, pooled: bool = False) -> None:
    """g = dy * relu6'(a*scale + shift) and the BatchNorm-backward sums of g.  pooled: dy is the
    (N, 1, 1, C) gradient of the average pool over a's H*W pixels, spread as dy / (H*W)."""
    N, H, W, Cc = a.shape
    if pooled:
        assert tuple(dy.shape) == (N, 1, 1, Cc)
    check(lib().atomai_b200_relu6_bwd_reduce(ptr(dy), _ld(dy), ptr(a), _ld(a), ptr(scale),
                                             ptr(shift), ptr(mean), ptr(invstd), ptr(g), _ld(g),
                                             N * H * W, Cc, H * W if pooled else 0, ptr(sums),
                                             stream_ptr()))


def affine_relu6(a, scale, shift, y) -> None:
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_affine_relu6(ptr(a), _ld(a), ptr(scale), ptr(shift), ptr(y), _ld(y),
                                         N * H * W, Cc, stream_ptr()))


def avgpool_relu6_fwd(a, scale, shift, y) -> None:
    """y (N, C) = AdaptiveAvgPool2d(1) of relu6(a*scale + shift)."""
    N, H, W, Cc = a.shape
    assert y.is_contiguous() and y.numel() == N * Cc
    check(lib().atomai_b200_avgpool_relu6_fwd(ptr(a), _ld(a), ptr(scale), ptr(shift), ptr(y), N,
                                              H * W, Cc, stream_ptr()))


def avgpool_bwd(dy, g) -> None:
    N, H, W, Cc = g.shape
    assert dy.is_contiguous() and dy.numel() == N * Cc
    check(lib().atomai_b200_avgpool_bwd(ptr(dy), ptr(g), _ld(g), N, H * W, Cc, stream_ptr()))


def log_softmax_fwd(x, y) -> None:
    B, Cc = x.shape
    assert x.is_contiguous() and y.is_contiguous()
    check(lib().atomai_b200_log_softmax_fwd(ptr(x), ptr(y), B, Cc, stream_ptr()))


def log_softmax_bwd(y, dy, dx) -> None:
    B, Cc = y.shape
    assert y.is_contiguous() and dy.is_contiguous() and dx.is_contiguous()
    check(lib().atomai_b200_log_softmax_bwd(ptr(y), ptr(dy), ptr(dx), B, Cc, stream_ptr()))


def nll_fwd_bwd(logp, target, loss=None, dlogp=None, gscale_dev=None) -> None:
    B, Cc = logp.shape
    assert logp.is_contiguous() and target.dtype == torch.int64 and target.is_contiguous()
    assert target.numel() == B
    check(lib().atomai_b200_nll_fwd_bwd(ptr(logp), ptr(target), B, Cc, ptr(loss), ptr(dlogp),
                                        ptr(gscale_dev), stream_ptr()))


def transpose(x, y, N, R, Cc) -> None:
    """y[n][c][r] = x[n][r][c] (both contiguous)."""
    assert x.is_contiguous() and y.is_contiguous() and x.numel() == y.numel() == N * R * Cc
    check(lib().atomai_b200_transpose(ptr(x), ptr(y), N, R, Cc, stream_ptr()))


def add_slice(src, dst, accumulate) -> None:
    N, H, W, Cc = src.shape
    check(lib().atomai_b200_add_slice(ptr(src), _ld(src), ptr(dst), _ld(dst),
                                      1 if accumulate else 0, N * H * W, Cc, stream_ptr()))


def dilated_sum(a_list, scale_list, shift_list, slope, out) -> None:
    # the kernel reads every layer and writes `out` as dense arrays of out.numel() elements
    assert out.is_contiguous() and all(t.is_contiguous() and t.numel() == out.numel()
                                       for t in a_list), "dilated_sum: dense tensors expected"
    n = len(a_list)
    arr = C.c_void_p * n
    a = arr(*[t.data_ptr() for t in a_list])
    sc = arr(*[ptr(t) for t in scale_list])
    sh = arr(*[ptr(t) for t in shift_list])
    check(lib().atomai_b200_dilated_sum(a, sc, sh, n, float(slope), ptr(out), out.numel(),
                                        out.shape[-1], stream_ptr()))


def ce_fwd_bwd(logits_nhwc, labels, loss_sum, dlogits=None, gscale=1.0, gscale_dev=None) -> None:
    N, H, W, Cc = logits_nhwc.shape
    assert labels.dtype == torch.int64 and labels.is_contiguous()
    check(lib().atomai_b200_ce_fwd_bwd(ptr(logits_nhwc), _ld(logits_nhwc), ptr(labels),
                                       N * H * W, Cc, ptr(loss_sum), ptr(dlogits),
                                       _ld(dlogits) if dlogits is not None else 0, float(gscale),
                                       ptr(gscale_dev), stream_ptr()))


def pointwise_loss(pred, target, kind, loss_sum, dpred=None, gscale=1.0, gscale_dev=None) -> None:
    assert pred.is_contiguous() and target.is_contiguous() and pred.numel() == target.numel()
    check(lib().atomai_b200_pointwise_loss(ptr(pred), ptr(target), pred.numel(), kind,
                                           ptr(loss_sum), ptr(dpred), float(gscale),
                                           ptr(gscale_dev), stream_ptr()))


def _labels(labels) -> int:
    """label_float flag of the segmentation objectives (float labels are truncated, int64 read)."""
    assert labels.is_cuda and labels.is_contiguous() and labels.dtype in (torch.int64, torch.float32)
    return 1 if labels.dtype == torch.float32 else 0


def dice_sums(logits_nhwc, labels, cells) -> None:
    """cells (float64, 2K) <- per-cell (I, S) sums of the dice loss (K = C*W, or 2 for C == 1)."""
    N, H, W, Cc = logits_nhwc.shape
    assert cells.dtype == torch.float64 and cells.is_contiguous() and labels.numel() == N * H * W
    check(lib().atomai_b200_dice_sums(ptr(logits_nhwc), _ld(logits_nhwc), ptr(labels),
                                      _labels(labels), N, H, W, Cc, ptr(cells), stream_ptr()))


def dice_finalize(cells, eps, loss, coef=None) -> None:
    check(lib().atomai_b200_dice_finalize(ptr(cells), cells.numel() // 2, float(eps), ptr(loss),
                                          ptr(coef), stream_ptr()))


def dice_bwd(logits_nhwc, labels, coef, dlogits, gscale=1.0, gscale_dev=None) -> None:
    N, H, W, Cc = logits_nhwc.shape
    check(lib().atomai_b200_dice_bwd(ptr(logits_nhwc), _ld(logits_nhwc), ptr(labels),
                                     _labels(labels), N, H, W, Cc, ptr(coef), ptr(dlogits),
                                     _ld(dlogits), float(gscale), ptr(gscale_dev), stream_ptr()))


def focal_finalize(bce_sum, count, alpha, gamma, loss, factor=None) -> None:
    check(lib().atomai_b200_focal_finalize(ptr(bce_sum), float(count), float(alpha), float(gamma),
                                           ptr(loss), ptr(factor), stream_ptr()))


def iou_hist(logits_nhwc, labels, thresh, counts, activation=True) -> None:
    """counts (int64, nc*nc, zeroed) += confusion histogram of thresholded predictions vs labels
    (softmax / sigmoid applied first unless `activation` is false)."""
    N, H, W, Cc = logits_nhwc.shape
    assert counts.dtype == torch.int64 and counts.is_contiguous() and labels.numel() == N * H * W
    check(lib().atomai_b200_iou_hist(ptr(logits_nhwc), _ld(logits_nhwc), ptr(labels),
                                     _labels(labels), N * H * W, Cc, 1 if activation else 0,
                                     float(thresh), ptr(counts),
                                     stream_ptr()))


def iou_finalize(counts, nc, out) -> None:
    check(lib().atomai_b200_iou_finalize(ptr(counts), int(nc), ptr(out), stream_ptr()))


def sqerr_reduce(x, xhat, out, dxhat=None, gscale=1.0, gscale_dev=None) -> None:
    check(lib().atomai_b200_sqerr_reduce(ptr(x), ptr(xhat), x.numel(), ptr(out), ptr(dxhat),
                                         float(gscale), ptr(gscale_dev), stream_ptr()))


def adam_multi(table_dev, n, max_numel, lr, b1, b2, eps, wd, step, grad_scale=1.0) -> None:
    check(lib().atomai_b200_adam_multi(ptr(table_dev), n, max_numel, lr, b1, b2, eps, wd, step,
                                       grad_scale, stream_ptr()))


def gemm(A, a_sm, a_sk, B, b_sk, b_sn, Cm, c_sm, M, N, K, bias=None, act=ACT_LRELU, slope=1.0,
         accumulate=False, split_k=1) -> None:
    check(lib().atomai_b200_gemm(ptr(A), a_sm, a_sk, ptr(B), b_sk, b_sn, ptr(Cm), c_sm, M, N, K,
                                 ptr(bias), act, float(slope), 1 if accumulate else 0, split_k,
                                 stream_ptr()))


def linear_fwd(x, w, b, y) -> None:
    Bn, K = x.shape
    O = w.shape[0]
    check(lib().atomai_b200_linear_fwd(ptr(x), ptr(w), ptr(b), ptr(y), Bn, K, O, stream_ptr()))


def linear_bwd(x, w, dy, dx, dw, db) -> None:
    Bn, K = x.shape
    O = w.shape[0]
    check(lib().atomai_b200_linear_bwd(ptr(x), ptr(w), ptr(dy), ptr(dx), ptr(dw), ptr(db), Bn, K,
                                       O, stream_ptr()))


def coord_latent_desc(B, H, W, z, phi, dx, wc, bc, wz, tanh_act) -> _C.CoordLat:
    d = _C.CoordLat()
    d.B, d.H, d.W, d.zdim, d.hid, d.tanh_act = B, H, W, (z.shape[1] if z is not None else 0), \
        wc.shape[0], 1 if tanh_act else 0
    d.z, d.phi, d.dx, d.wc, d.bc, d.wz = ptr(z), ptr(phi), ptr(dx), ptr(wc), ptr(bc), ptr(wz)
    return d


def coord_latent_fwd(d: _C.CoordLat, h0) -> None:
    check(lib().atomai_b200_coord_latent_fwd(C.byref(d), ptr(h0), stream_ptr()))


def coord_latent_bwd(d: _C.CoordLat, dpre0, dwc, dbc, sb, dphi, ddx) -> None:
    check(lib().atomai_b200_coord_latent_bwd(C.byref(d), ptr(dpre0), ptr(dwc), ptr(dbc), ptr(sb),
                                             ptr(dphi), ptr(ddx), stream_ptr()))


def jlat_desc(B, Dc, coord, heads, tau, phi_prior=0.1, dx_prior=0.1) -> _C.JLat:
    """Descriptor of the joint latent block: B rows, Dc continuous columns (coord of them rotation /
    translation), discrete heads of sizes `heads`, Gumbel-softmax temperature tau."""
    if not 1 <= len(heads) <= _C.JLAT_MAX_DISC:
        raise ValueError(f"joint latent: {len(heads)} discrete heads (1..{_C.JLAT_MAX_DISC})")
    d = _C.JLat()
    d.B, d.Dc, d.coord, d.nheads = int(B), int(Dc), int(coord), len(heads)
    for i, h in enumerate(heads):
        d.heads[i] = int(h)
    d.tau, d.phi_prior, d.dx_prior = float(tau), float(phi_prior), float(dx_prior)
    return d


def _check_args(status: int) -> None:
    """check() for entry points whose failures are arguments outside their documented limits."""
    try:
        check(status)
    except _C.NativeError as e:
        raise ValueError(str(e)) from None


def jlatent_fwd(d: _C.JLat, mode: int, mu, logsd, logits, eps, u, seed: int, alpha, zdec=None,
                phi=None, dx=None, kl=None) -> None:
    """alpha (B, D) <- head softmax of logits; mode JLAT_SAMPLE also writes the decoder input zdec,
    phi / dx (coord > 0) and kl = [continuous KL mean, discrete KL sum of means] (nullable).  The
    Gumbel noise comes from `u` (B, D) when given, else from the hash generator with `seed`."""
    _check_args(lib().atomai_b200_jlatent_fwd(
        C.byref(d), mode, ptr(mu), ptr(logsd), ptr(logits), ptr(eps), ptr(u), int(seed) & (2**64 - 1),
        ptr(alpha), ptr(zdec), ptr(phi), ptr(dx), ptr(kl), stream_ptr()))


def jlatent_bwd(d: _C.JLat, mode: int, mu, logsd, logits, eps, u, seed: int, dzdec, dphi, ddx,
                dalpha, gkl, dmu, dlogsd, dlogits) -> None:
    """Gradients of jlatent_fwd w.r.t. mu, logsd and logits (every incoming gradient nullable)."""
    _check_args(lib().atomai_b200_jlatent_bwd(
        C.byref(d), mode, ptr(mu), ptr(logsd), ptr(logits), ptr(eps), ptr(u), int(seed) & (2**64 - 1),
        ptr(dzdec), ptr(dphi), ptr(ddx), ptr(dalpha), ptr(gkl), ptr(dmu), ptr(dlogsd), ptr(dlogits),
        stream_ptr()))


def gram(x1, x2, inv_ls, outputscale, kind, out, math=MATH_TF32X3) -> None:
    n1, d = x1.shape
    n2 = x2.shape[0]
    nbytes = lib().atomai_b200_gram_workspace_bytes(n1, n2, d)
    ws = torch.empty(nbytes + 256, device=x1.device, dtype=torch.uint8)
    off = (-ws.data_ptr()) % 256
    check(lib().atomai_b200_gram(ptr(x1), ptr(x2), ptr(inv_ls), float(outputscale), n1, n2, d,
                                 kind, math, ptr(out), out.stride(0), ws.data_ptr() + off, nbytes,
                                 stream_ptr()))


def gram_matvec(xq, x, inv_ls, alpha, c, outputscale, kind, out) -> None:
    """out[i] = c + outputscale * sum_j k(||(xq_i - x_j) * inv_ls||) alpha_j without forming the
    cross-Gram: xq (nq, d), x (n, d), inv_ls (d,) fp32; alpha (n,), out (nq,) float64; d <= 4."""
    nq, d = xq.shape
    n = x.shape[0]
    assert xq.dtype == x.dtype == inv_ls.dtype == torch.float32 and x.shape[1] == d
    assert alpha.dtype == out.dtype == torch.float64 and alpha.numel() == n and out.numel() == nq
    assert all(t.is_contiguous() for t in (xq, x, inv_ls, alpha, out)) and inv_ls.numel() == d
    check(lib().atomai_b200_gram_matvec(ptr(xq), ptr(x), ptr(inv_ls), ptr(alpha), float(c),
                                        float(outputscale), nq, n, d, kind, ptr(out),
                                        stream_ptr()))


def gram_f64(x, inv_ls, outputscale, noise, kind, out) -> None:
    """out (n, n) float64 <- outputscale * k(||(x_i - x_j) * inv_ls||) + noise on the diagonal;
    x (n, d) and inv_ls (d,) float64, d <= 4."""
    n, d = x.shape
    assert x.dtype == inv_ls.dtype == out.dtype == torch.float64 and inv_ls.numel() == d
    assert x.is_contiguous() and inv_ls.is_contiguous() and out.shape == (n, n) and out.stride(1) == 1
    check(lib().atomai_b200_gram_f64(ptr(x), ptr(inv_ls), float(outputscale), float(noise), n, d,
                                     kind, ptr(out), out.stride(0), stream_ptr()))


def gram_f64_adjoint(x, inv_ls, kind, G, out) -> None:
    """out (d + 2,) float64 <- [sum G m t_k^2 (k < d), sum G k, trace G] for the Gram of gram_f64
    at unit outputscale (see include/atomai_b200.h)."""
    n, d = x.shape
    assert G.dtype == out.dtype == torch.float64 and G.shape == (n, n) and G.stride(1) == 1
    assert x.is_contiguous() and inv_ls.is_contiguous() and out.numel() == d + 2
    check(lib().atomai_b200_gram_f64_adjoint(ptr(x), ptr(inv_ls), n, d, kind, ptr(G), G.stride(0),
                                             ptr(out), stream_ptr()))


def prob_mask(logits_nhwc, mode: int, thresh: float, prob, mask=None) -> None:
    """prob = softmax (mode 0) / sigmoid (1) / exp (2) / identity (3) of NHWC logits; mask (uint8,
    optional) = prob > thresh."""
    N, H, W, Cc = logits_nhwc.shape
    assert prob.is_contiguous() and prob.shape == logits_nhwc.shape
    assert mask is None or (mask.dtype == torch.uint8 and mask.is_contiguous())
    check(lib().atomai_b200_prob_mask(ptr(logits_nhwc), _ld(logits_nhwc), N * H * W, Cc, mode,
                                      float(thresh), ptr(prob), Cc, ptr(mask), stream_ptr()))


def gather_windows(img_nhwc, table, r: int, out, nanflag=None) -> None:
    """out[k] = img[f, sx:sx+r, sy:sy+r, :] for the int32 rows (f, sx, sy) of `table`."""
    n, h, w, c = img_nhwc.shape
    assert img_nhwc.is_contiguous() and table.dtype == torch.int32 and table.is_contiguous()
    check(lib().atomai_b200_gather_windows(ptr(img_nhwc), n, h, w, c, ptr(table), table.shape[0], r,
                                           ptr(out), ptr(nanflag), stream_ptr()))


def gather_patches(img, offs, ph: int, pw: int, out) -> None:
    """out[k] = the ph x pw window at element offset offs[k] (int64) of a contiguous image whose last
    two dims are (w, c), as a bit copy; img and out share a dtype of 1, 2, 4 or 8 bytes."""
    w, c = img.shape[-2:]
    assert img.is_contiguous() and out.is_contiguous() and img.dtype == out.dtype
    assert offs.dtype == torch.int64 and offs.is_contiguous() and out.numel() == offs.numel() * ph * pw * c
    check(lib().atomai_b200_gather_patches(ptr(img), img.element_size(), w, c, ptr(offs),
                                           offs.shape[0], ph, pw, ptr(out), stream_ptr()))


def imgen_masks(atoms, frames, max_pix: int, owner, tpl, out, background: bool) -> None:
    """Lattice masks: the owner pass over the int32 atom rows, then the fill pass (see
    include/atomai_b200.h); `owner` must be zeroed, `tpl` and `out` share a dtype."""
    assert atoms.dtype == owner.dtype == torch.int32 and frames.dtype == torch.int64
    assert atoms.shape[1:] == (_C.IMGEN_ATOM_INTS,) and frames.shape[1:] == (_C.IMGEN_FRAME_INTS,)
    assert all(t.is_contiguous() for t in (atoms, frames, owner, tpl, out)) and tpl.dtype == out.dtype
    check(lib().atomai_b200_imgen_owner(ptr(atoms), atoms.shape[0], ptr(frames), ptr(owner),
                                        stream_ptr()))
    check(lib().atomai_b200_imgen_fill(ptr(atoms), ptr(frames), frames.shape[0], max_pix,
                                       ptr(owner), ptr(tpl), out.element_size(), int(background),
                                       ptr(out), stream_ptr()))


BLOB_CODES = {torch.uint8: _C.BLOB_U8, torch.int16: _C.BLOB_I16, torch.uint16: _C.BLOB_U16,
              torch.float32: _C.BLOB_F32, torch.float64: _C.BLOB_F64, torch.int32: _C.BLOB_I32}


def blob_filter(img, im_thresh: float, blob_thresh: float, above: bool, labels, counts,
                out) -> None:
    """Threshold, 4-connected labelling and size filter of every frame of the (n, h, w) stack
    `img` into `out` (see include/atomai_b200.h); `labels` and `counts` are (n, h, w) int32
    workspaces, left holding each pixel's smallest component index and the component sizes."""
    assert img.dim() == 3 and img.dtype in BLOB_CODES and img.dtype != torch.int32
    assert labels.dtype == counts.dtype == torch.int32 and out.dtype in BLOB_CODES
    assert labels.shape == counts.shape == out.shape == img.shape
    assert all(t.is_contiguous() for t in (img, labels, counts, out))
    n, h, w = img.shape
    check(lib().atomai_b200_blob_filter(ptr(img), BLOB_CODES[img.dtype], n, h, w, im_thresh,
                                        blob_thresh, int(above), ptr(labels), ptr(counts),
                                        ptr(out), BLOB_CODES[out.dtype], stream_ptr()))


FFT_CODES = {torch.uint8: _C.FFT_U8, torch.bool: _C.FFT_U8, torch.int8: _C.FFT_I8,
             torch.int16: _C.FFT_I16, torch.uint16: _C.FFT_U16, torch.int32: _C.FFT_I32,
             torch.uint32: _C.FFT_U32, torch.int64: _C.FFT_I64, torch.uint64: _C.FFT_U64,
             torch.float16: _C.FFT_F16, torch.float32: _C.FFT_F32, torch.float64: _C.FFT_F64,
             torch.complex64: _C.FFT_C64, torch.complex128: _C.FFT_C128}


def fft2_workspace_bytes(h: int, w: int) -> int:
    """bytes of device scratch fft2_mask / fft2_sub need for an (h, w) array (-1: side too long)"""
    return int(lib().atomai_b200_fft2_workspace_bytes(h, w))


def _fft2_work(h: int, w: int):
    n = fft2_workspace_bytes(h, w)
    assert n > 0, (h, w)
    return torch.empty(n, dtype=torch.uint8, device="cuda"), n


def fft2_mask(img, r0: int, c0: int, l: int, f2, f3) -> None:
    """f2 = fftshift(fft2(img)) and f3 = f2 with the disk of half-width l at (r0, c0) zeroed, both
    (h, w) complex64 or complex128, from a float64 transform (see include/atomai_b200.h)"""
    assert img.dim() == 2 and img.dtype in FFT_CODES and img.is_contiguous()
    assert f2.dtype == f3.dtype and f2.dtype in (torch.complex64, torch.complex128)
    assert f2.shape == f3.shape == img.shape and f2.is_contiguous() and f3.is_contiguous()
    h, w = img.shape
    work, nbytes = _fft2_work(h, w)
    check(lib().atomai_b200_fft2_mask(ptr(img), FFT_CODES[img.dtype], h, w, r0, c0, l, ptr(f2),
                                      ptr(f3), int(f2.dtype == torch.complex64), ptr(work),
                                      nbytes, stream_ptr()))


def fft2_sub(img, spec, out) -> None:
    """out = min-max normalised |img - Re(ifft2(ifftshift(spec)))|, float32 or float64, computed
    in float64 (see include/atomai_b200.h)"""
    assert img.dim() == 2 and img.dtype in FFT_CODES and img.is_contiguous()
    assert spec.dtype in (torch.complex64, torch.complex128) and spec.is_contiguous()
    assert out.dtype in (torch.float32, torch.float64) and out.is_contiguous()
    assert spec.shape == out.shape == img.shape
    h, w = img.shape
    work, nbytes = _fft2_work(h, w)
    check(lib().atomai_b200_fft2_sub(ptr(img), FFT_CODES[img.dtype], ptr(spec),
                                     FFT_CODES[spec.dtype], h, w, ptr(out),
                                     int(out.dtype == torch.float32), ptr(work), nbytes,
                                     stream_ptr()))


STAT_GMM, STAT_KMEANS, STAT_KPP = 0, 1, 2


def _stat_math(math):
    from .engine import _MATH
    return _MATH["mode"] if math is None else math


def stat_estep(X, mu, mode, A, B, cst, out, closest=None, resp=None, labels=None, rowval=None,
               D=None, changes=None, math=None) -> None:
    """One pass over the fp32 (N, d) X centred by mu: GMM responsibilities / k-means assignment /
    k-means++ candidate potentials (see include/atomai_b200.h); out is float64.  `math`
    (MATH_*, default: the set_math mode) picks the wgmma or the exact-FFMA kernel."""
    N, d = X.shape
    K = A.shape[0]
    assert X.is_contiguous() and X.dtype == torch.float32 and A.shape == (K, d)
    assert out.dtype == torch.float64
    check(lib().atomai_b200_stat_estep(ptr(X), ptr(mu), N, d, K, mode, ptr(A), ptr(B), ptr(cst),
                                       ptr(closest), ptr(resp), ptr(labels), ptr(rowval), ptr(D),
                                       ptr(out), ptr(changes), _stat_math(math), stream_ptr()))


def stat_accum(X, mu, K, sx, sxx=None, nk=None, resp=None, labels=None, math=None) -> None:
    """float64 sx (K, d) = sum_n r_nk (x_n - mu), sxx likewise of the squares, nk = sum_n r_nk, with
    r = resp (N, K) fp32, else one-hot int32 labels, else all rows in component 0; `math` as in
    stat_estep."""
    N, d = X.shape
    assert X.is_contiguous() and X.dtype == torch.float32 and sx.shape == (K, d)
    check(lib().atomai_b200_stat_accum(ptr(X), ptr(mu), N, d, K, ptr(resp), ptr(labels), ptr(sx),
                                       ptr(sxx), ptr(nk), _stat_math(math), stream_ptr()))


def stat_gmm_params(sx, sxx, nk, N, spherical, reg_covar, init, means, covs, weights, A, B, cst):
    K, d = sx.shape
    check(lib().atomai_b200_stat_gmm_params(ptr(sx), ptr(sxx), ptr(nk), N, d, K, int(spherical),
                                            float(reg_covar), int(init), ptr(means), ptr(covs),
                                            ptr(weights), ptr(A), ptr(B), ptr(cst), stream_ptr()))


def stat_kmeans_centres(c_new, A, cst, sx=None, nk=None, c_old=None, shift=None) -> None:
    K, d = c_new.shape
    check(lib().atomai_b200_stat_kmeans_centres(ptr(sx), ptr(nk), ptr(c_old), ptr(c_new), K, d,
                                                ptr(A), ptr(cst), ptr(shift), stream_ptr()))


def stat_kpp_chunks(N: int) -> int:
    return int(lib().atomai_b200_stat_kpp_chunks(N))


def stat_kpp_candidates(closest, N, ntr, seed, counter, chunk_ws, idx) -> None:
    check(lib().atomai_b200_stat_kpp_candidates(ptr(closest), N, ntr, seed, counter, ptr(chunk_ws),
                                                ptr(idx), stream_ptr()))


def stat_gather_rows(X, mu, idx, out) -> None:
    check(lib().atomai_b200_stat_gather_rows(ptr(X), ptr(mu), X.shape[1], ptr(idx), idx.numel(),
                                             ptr(out), stream_ptr()))


def stat_kpp_commit(D, pot, closest, cand, centre) -> None:
    N, ntr = D.shape
    check(lib().atomai_b200_stat_kpp_commit(ptr(D), ntr, ptr(pot), ptr(closest), N, ptr(cand),
                                            cand.shape[1], ptr(centre), stream_ptr()))


DECOMP_MAX_K = 64      # components per decomp_project call and limit of the NMF / FastICA passes


def decomp_slot_doubles(op: int, N: int, d: int, K: int) -> int:
    """ordered-slot workspace (doubles) of a decomp pass: op 0 / 1 gram (rows = op), 2 nmf_w,
    3 nmf_h, 4 ica_step"""
    return int(lib().atomai_b200_decomp_slot_doubles(op, N, d, K))


def decomp_gram(X, mu, G, rows: bool) -> None:
    """float64 G = (X - mu)^T (X - mu) (d x d), or (X - mu)(X - mu)^T (N x N) when `rows`; mu
    (d,) fp32 or None.  Exact fp32 FFMA whatever set_math says."""
    N, d = X.shape
    m = N if rows else d
    assert X.is_contiguous() and X.dtype == torch.float32
    assert G.dtype == torch.float64 and G.shape == (m, m) and G.is_contiguous()
    check(lib().atomai_b200_decomp_gram(ptr(X), ptr(mu), N, d, int(rows), ptr(G), stream_ptr()))


def decomp_project(X, mu, B, out) -> None:
    """fp32 out (N, k) = (X - mu) B^T for B (k, d), any k (blocks of DECOMP_MAX_K rows of B)."""
    N, d = X.shape
    k = B.shape[0]
    assert X.is_contiguous() and X.dtype == B.dtype == out.dtype == torch.float32
    assert B.shape == (k, d) and B.is_contiguous() and out.shape == (N, k) and out.is_contiguous()
    for k0 in range(0, k, DECOMP_MAX_K):
        kb = min(DECOMP_MAX_K, k - k0)
        check(lib().atomai_b200_decomp_project(ptr(X), ptr(mu), N, d, kb, B[k0].data_ptr(),
                                               out[:, k0].data_ptr(), k, stream_ptr()))


def decomp_nmf_w(X, H, HHt, W, out) -> None:
    """one coordinate-descent sweep of W (N, k) in place; out (k * k + 1,) float64 <- [W^T W,
    violation]"""
    N, d = X.shape
    k = H.shape[0]
    assert X.dtype == H.dtype == W.dtype == torch.float32 and HHt.dtype == out.dtype == torch.float64
    assert W.shape == (N, k) and H.shape == (k, d) and HHt.shape == (k, k) and out.numel() == k * k + 1
    assert all(t.is_contiguous() for t in (X, H, HHt, W, out))
    check(lib().atomai_b200_decomp_nmf_w(ptr(X), N, d, k, ptr(H), ptr(HHt), ptr(W), ptr(out),
                                         stream_ptr()))


def decomp_nmf_h(WtX, WtW, H, out) -> None:
    """one coordinate-descent sweep of H (k, d) in place from W^T X (k, d) and W^T W (float64);
    out (k * k + 1,) float64 <- [H H^T, violation]"""
    k, d = H.shape
    assert H.dtype == torch.float32 and WtX.dtype == WtW.dtype == out.dtype == torch.float64
    assert WtX.shape == (k, d) and WtW.shape == (k, k) and out.numel() == k * k + 1
    assert all(t.is_contiguous() for t in (WtX, WtW, H, out))
    check(lib().atomai_b200_decomp_nmf_h(ptr(WtX), ptr(WtW), d, k, ptr(H), ptr(out), stream_ptr()))


def decomp_ica_step(X1, W, out) -> None:
    """FastICA pass over the whitened samples X1 (N, k) fp32 with W (k, k) float64: out (k * k + k,)
    float64 <- [sum_n tanh(W x_n) x_n^T, sum_n (1 - tanh(W x_n)^2)]"""
    N, k = X1.shape
    assert X1.dtype == torch.float32 and W.dtype == out.dtype == torch.float64
    assert W.shape == (k, k) and out.numel() == k * k + k
    assert all(t.is_contiguous() for t in (X1, W, out))
    check(lib().atomai_b200_decomp_ica_step(ptr(X1), N, k, ptr(W), ptr(out), stream_ptr()))


def _grid_args(lo, dims):
    return (C.c_double * 3)(*[float(v) for v in lo]), (C.c_int64 * 3)(*[int(v) for v in dims])


def graph_cell_keys(pos, frame, lo, side: float, dims, keys) -> None:
    """int64 cell key of every atom of pos (N, 3) float64: ((frame * nz + cz) * ny + cy) * nx + cx
    for cells of side `side` from the origin lo (3 floats), dims = (nx, ny, nz); frame (N,) int32
    or None."""
    N = pos.shape[0]
    assert pos.dtype == torch.float64 and pos.shape == (N, 3) and pos.is_contiguous()
    assert keys.dtype == torch.int64 and keys.shape == (N,)
    assert frame is None or (frame.dtype == torch.int32 and frame.shape == (N,))
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_graph_cell_keys(ptr(pos), ptr(frame), N, lo_, float(side), dims_,
                                            ptr(keys), stream_ptr()))


def graph_bonds(pos, cls, frame, keys, perm, cut, lo, side: float, dims, rowptr, out) -> None:
    """Bonds within the C x C float64 cutoff table `cut` (class pair of cls, (N,) int32 or None).
    keys / perm: the sorted cell keys and the atom of each.  rowptr None: out (N,) int32 = degrees;
    else out[rowptr[i]:rowptr[i + 1]] = the atoms bonded to i, ascending."""
    N = pos.shape[0]
    Cn = cut.shape[0]
    assert pos.dtype == cut.dtype == torch.float64 and pos.shape == (N, 3) and pos.is_contiguous()
    assert cut.shape == (Cn, Cn) and cut.is_contiguous()
    assert keys.dtype == perm.dtype == torch.int64 and keys.shape == perm.shape == (N,)
    assert cls is None or (cls.dtype == torch.int32 and cls.shape == (N,))
    assert frame is None or (frame.dtype == torch.int32 and frame.shape == (N,))
    assert out.dtype == torch.int32 and (rowptr is not None or out.shape == (N,))
    assert rowptr is None or (rowptr.dtype == torch.int64 and rowptr.shape == (N + 1,))
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_graph_bonds(ptr(pos), ptr(cls), ptr(frame), N, ptr(keys), ptr(perm),
                                        ptr(cut), Cn, lo_, float(side), dims_, ptr(rowptr),
                                        ptr(out), stream_ptr()))


def graph_hops(rowptr, cols, bptr, ball, optr, out, cnt) -> None:
    """One level of the packed (id << 5 | hops) hop table: optr None: cnt (N,) int64 = row lengths
    of the next level; else out[optr[u]:optr[u + 1]] = u's next-level row."""
    N = rowptr.shape[0] - 1
    assert rowptr.dtype == bptr.dtype == torch.int64 and bptr.shape == (N + 1,)
    assert cols.dtype == torch.int32 and ball.dtype == torch.int32
    assert optr is None or (out is not None and out.dtype == torch.int32 and optr.shape == (N + 1,))
    assert optr is not None or (cnt.dtype == torch.int64 and cnt.shape == (N,))
    check(lib().atomai_b200_graph_hops(ptr(rowptr), ptr(cols), N, ptr(bptr), ptr(ball), ptr(optr),
                                       ptr(out), ptr(cnt), stream_ptr()))


def graph_rings(rowptr, cols, bptr, ball, max_depth: int, ring_base=None, atom_base=None,
                lens=None, atoms=None, cnt=None) -> None:
    """Rings of 3 ... max_depth atoms, one search per root atom.  ring_base None: cnt (N, 3) int64
    = (rings, ring atoms, search steps) per root; else the rings of root r go to
    lens[ring_base[r]:] and atoms[atom_base[r]:] (int32) in discovery order."""
    N = rowptr.shape[0] - 1
    assert rowptr.dtype == bptr.dtype == torch.int64 and bptr.shape == (N + 1,)
    assert cols.dtype == torch.int32 and ball.dtype == torch.int32
    if ring_base is None:
        assert cnt.dtype == torch.int64 and cnt.shape == (N, 3) and cnt.is_contiguous()
    else:
        assert ring_base.dtype == atom_base.dtype == torch.int64 and ring_base.shape == (N,)
        assert lens.dtype == atoms.dtype == torch.int32
    check(lib().atomai_b200_graph_rings(ptr(rowptr), ptr(cols), N, ptr(bptr), ptr(ball),
                                        int(max_depth), ptr(ring_base), ptr(atom_base), ptr(lens),
                                        ptr(atoms), ptr(cnt), stream_ptr()))


def graph_ring_filter(off, lens, atoms, bptr, ball, keep) -> None:
    """keep (R,) uint8: 0 for the rings with a shortcut through the bond graph, else 1."""
    R = lens.shape[0]
    assert off.dtype == bptr.dtype == torch.int64 and off.shape == (R,)
    assert lens.dtype == atoms.dtype == ball.dtype == torch.int32
    assert keep.dtype == torch.uint8 and keep.shape == (R,)
    check(lib().atomai_b200_graph_ring_filter(ptr(off), ptr(lens), ptr(atoms), R, ptr(bptr),
                                              ptr(ball), ptr(keep), stream_ptr()))


def coords_cells(pos, lo, side: float, dims, cells) -> None:
    """cells (N, 3) int64: the grid cell of every row of pos (N, 3) float64, as graph_cell_keys
    bins it."""
    N = pos.shape[0]
    assert pos.dtype == torch.float64 and pos.shape == (N, 3) and pos.is_contiguous()
    assert cells.dtype == torch.int64 and cells.shape == (N, 3) and cells.is_contiguous()
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_coords_cells(ptr(pos), N, lo_, float(side), dims_, ptr(cells),
                                         stream_ptr()))


def coords_knn(qpos, qcell, qframe, pos, keys, perm, foff, lo, side: float, dims, k: int,
               ub: float, oidx, odist) -> None:
    """The k nearest rows of pos (N, 3) float64 with distance < ub to every query (qpos (Q, 3),
    in cells qcell (Q, 3) int64), within the query's frame qframe (Q,) int32 whose atoms are the
    sorted keys foff[f]:foff[f + 1] (both None: one frame).  oidx (Q, k) int32 / odist (Q, k)
    float64 ascending, -1 / inf where fewer are found; an equal distance goes to the lower index."""
    Q, N = qpos.shape[0], pos.shape[0]
    assert qpos.dtype == pos.dtype == odist.dtype == torch.float64
    assert qpos.shape == (Q, 3) and pos.shape == (N, 3) and qpos.is_contiguous() and pos.is_contiguous()
    assert qcell.dtype == torch.int64 and qcell.shape == (Q, 3) and qcell.is_contiguous()
    assert keys.dtype == perm.dtype == torch.int64 and keys.shape == perm.shape == (N,)
    assert (qframe is None) == (foff is None)
    assert qframe is None or (qframe.dtype == torch.int32 and qframe.shape == (Q,)
                              and foff.dtype == torch.int64)
    assert oidx.dtype == torch.int32 and oidx.shape == odist.shape == (Q, k)
    assert oidx.is_contiguous() and odist.is_contiguous()
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_coords_knn(ptr(qpos), ptr(qcell), ptr(qframe), Q, ptr(pos), N,
                                       ptr(keys), ptr(perm), ptr(foff), lo_, float(side), dims_,
                                       int(k), float(ub), ptr(oidx), ptr(odist), stream_ptr()))


def coords_ball(qpos, qcell, pos, keys, perm, lo, side: float, dims, rmax: float, rowptr=None,
                oidx=None, odist=None, cnt=None) -> None:
    """Rows of pos with distance < rmax (<= side) of every query.  rowptr None: cnt (Q,) int64 =
    their number; else oidx (int32) / odist (float64)[rowptr[i]:rowptr[i + 1]] = them, in scan
    order."""
    Q, N = qpos.shape[0], pos.shape[0]
    assert qpos.dtype == pos.dtype == torch.float64 and qpos.shape == (Q, 3) and pos.shape == (N, 3)
    assert qpos.is_contiguous() and pos.is_contiguous()
    assert qcell.dtype == torch.int64 and qcell.shape == (Q, 3) and qcell.is_contiguous()
    assert keys.dtype == perm.dtype == torch.int64 and keys.shape == perm.shape == (N,)
    if rowptr is None:
        assert cnt.dtype == torch.int64 and cnt.shape == (Q,)
    else:
        assert rowptr.dtype == torch.int64 and rowptr.shape == (Q + 1,)
        assert oidx.dtype == torch.int32 and odist.dtype == torch.float64
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_coords_ball(ptr(qpos), ptr(qcell), Q, ptr(pos), N, ptr(keys), ptr(perm),
                                        lo_, float(side), dims_, float(rmax), ptr(rowptr), ptr(oidx),
                                        ptr(odist), ptr(cnt), stream_ptr()))


def coords_walk(start, scell, pos, pcell, keys, perm, foff, lo, side: float, dims, rmax: float,
                H: int, W: int, half: int, r: int, out) -> None:
    """One walk per start (S, 3) through the frames of pos (atoms of frame f: sorted keys
    foff[f]:foff[f + 1]): out (S, F, 4) int32 = (f, atom, row0, col0) of each step, or
    (f, -1, -1, -1) where the frame is skipped (no atom with d < rmax, or numpy's slice
    [cx - half : cx + half, cy - half : cy + half] of an H x W image is not r x r)."""
    S, N, F = start.shape[0], pos.shape[0], foff.shape[0] - 1
    assert start.dtype == pos.dtype == torch.float64 and start.shape == (S, 3) and pos.shape == (N, 3)
    assert scell.dtype == pcell.dtype == torch.int64 and scell.shape == (S, 3) and pcell.shape == (N, 3)
    assert keys.dtype == perm.dtype == foff.dtype == torch.int64 and keys.shape == perm.shape == (N,)
    assert out.dtype == torch.int32 and out.shape == (S, F, 4) and out.is_contiguous()
    lo_, dims_ = _grid_args(lo, dims)
    check(lib().atomai_b200_coords_walk(ptr(start), ptr(scell), S, ptr(pos), ptr(pcell), ptr(keys),
                                        ptr(perm), ptr(foff), F, lo_, float(side), dims_,
                                        float(rmax), int(H), int(W), int(half), int(r), ptr(out),
                                        stream_ptr()))


def coords_dbscan_roots(rowptr, cols, min_samples: int, parent, flag) -> None:
    """parent (N,) int32: the least core index of the component of every core point of the CSR
    neighbourhoods (row length + 1 >= min_samples), -1 for the others.  flag: 1 int32 scratch."""
    N = rowptr.shape[0] - 1
    assert rowptr.dtype == torch.int64 and cols.dtype == torch.int32
    assert parent.dtype == flag.dtype == torch.int32 and parent.shape == (N,)
    check(lib().atomai_b200_coords_dbscan_roots(ptr(rowptr), ptr(cols), N, int(min_samples),
                                                ptr(parent), ptr(flag), stream_ptr()))


def coords_dbscan_labels(rowptr, cols, parent, rank, labels) -> None:
    """labels (N,) int64 = rank[root] of every core point's root and of the least root among a
    border point's core neighbours, -1 for noise."""
    N = rowptr.shape[0] - 1
    assert rowptr.dtype == rank.dtype == labels.dtype == torch.int64 and cols.dtype == torch.int32
    assert parent.dtype == torch.int32 and parent.shape == rank.shape == labels.shape == (N,)
    check(lib().atomai_b200_coords_dbscan_labels(ptr(rowptr), ptr(cols), N, ptr(parent), ptr(rank),
                                                 ptr(labels), stream_ptr()))


def peak_refine(stack, atoms, dmax: int, popt, info, nfev=None) -> None:
    """One lmdif fit of a rotated 2-D Gaussian per int32 row (frame, row0, col0, d) of `atoms` to
    the windows of the fp32 (n, H, W) `stack`: popt (K, 7) float64, info / nfev (K,) int32."""
    n, h, w = stack.shape
    assert stack.dtype == torch.float32 and stack.is_contiguous()
    assert atoms.dtype == torch.int32 and atoms.is_contiguous() and atoms.shape[1:] == (4,)
    assert popt.dtype == torch.float64 and popt.is_contiguous() and info.dtype == torch.int32
    check(lib().atomai_b200_peak_refine(ptr(stack), n, h, w, ptr(atoms), atoms.shape[0], int(dmax),
                                        ptr(popt), ptr(info), ptr(nfev), stream_ptr()))


def rowloss(x, xhat, kind: int, out=None, dxhat=None, gvec=None) -> None:
    """Per-sample reconstruction loss over (B, D) rows (kind 0: 0.5*sum sq. err., 1: BCE logits)."""
    B = x.shape[0]
    D = x.numel() // max(B, 1)
    check(lib().atomai_b200_rowloss(ptr(x), ptr(xhat), B, D, kind, ptr(out), ptr(dxhat), ptr(gvec),
                                    stream_ptr()))


def dropout_(a, p: float, seed: int, stats=None) -> None:
    """In-place inverted dropout of an NHWC tensor (or gradient) from (seed, element index)."""
    N, H, W, Cc = a.shape
    check(lib().atomai_b200_dropout(ptr(a), _ld(a), N * H * W, Cc, float(p), int(seed) & (2**64 - 1),
                                    ptr(stats), stream_ptr()))


def augment(x, y, scratch, lab_in, lab_out, params, row_shift, in_min, in_max, seed, minmax) -> None:
    n, h, w = x.shape
    check(lib().atomai_b200_augment(ptr(x), ptr(y), ptr(scratch), ptr(lab_in), ptr(lab_out),
                                    ptr(params), ptr(row_shift), n, h, w, float(in_min),
                                    float(in_max), int(seed) & (2**64 - 1), ptr(minmax),
                                    stream_ptr()))


def selftest_tma(x, c0, w0, h0, n0, TWp, THp, swizzle_mode, smem_offset, out) -> None:
    N, H, W, Cc = x.shape
    check(lib().atomai_b200_selftest_tma(ptr(x), N, H, W, Cc, c0, w0, h0, n0, TWp, THp, swizzle_mode,
                                         smem_offset, ptr(out), stream_ptr()))
