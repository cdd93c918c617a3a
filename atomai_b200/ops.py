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


def transpose(x, y, N, R, Cc) -> None:
    """y[n][c][r] = x[n][r][c] (both contiguous)."""
    assert x.is_contiguous() and y.is_contiguous() and x.numel() == y.numel() == N * R * Cc
    check(lib().atomai_b200_transpose(ptr(x), ptr(y), N, R, Cc, stream_ptr()))


def add_slice(src, dst, accumulate) -> None:
    N, H, W, Cc = src.shape
    check(lib().atomai_b200_add_slice(ptr(src), _ld(src), ptr(dst), _ld(dst),
                                      1 if accumulate else 0, N * H * W, Cc, stream_ptr()))


def dilated_sum(a_list, scale_list, shift_list, slope, out) -> None:
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
