"""
Define-by-run native graph ("tape") that executes a network as a sequence of sm_90a kernels and
replays it backwards.  It is the host-side orchestration of the C ABI, not a compute path of its
own: torch supplies device memory, the current stream and the autograd *boundary* (one
torch.autograd.Function per network call); all arithmetic on activations happens in
libatomai_b200.so.

Key idea (SURVEY.md §7 H3, §2.4 K2-K5): an activation handle (`Act`) stores the post-activation,
pre-BatchNorm tensor `a` in NHWC together with a *pending* per-channel affine (the BatchNorm
normalisation) and a *pending* 2x2 max-pool.  Consumers apply both while loading their input, so
BatchNorm outputs, pooled tensors and torch.cat results are never written to HBM
(atomai/nets/fcnn.py:117-142 materialises all of them).
"""
import os
from typing import List, Optional, Sequence, Union

import torch

from . import ops
from .ops import ACT_LRELU, ACT_TANH, MATH_FP32, MATH_TF32, MATH_TF32X3, Source

_MATH = {"mode": MATH_TF32X3, "wgrad_tc": True,   # default: the mode that meets the fp32 tolerances
         "wgrad": MATH_TF32,                        # weight-gradient contraction (None: same mode)
         "fuse_up": False}                          # 2x upsampling on load (False: written out)


_MODES = {"fp32": MATH_FP32, "tf32": MATH_TF32, "tf32x3": MATH_TF32X3}
if os.environ.get("ATOMAI_B200_FUSE_UP", "0") == "1":     # A/B switch for benchmarking
    _MATH["fuse_up"] = True


_NO_POOLSTATS = os.environ.get("ATOMAI_B200_NO_POOLSTATS", "0") == "1"    # A/B switch (bring-up)


def set_fusion(upsample: Optional[bool] = None) -> None:
    """upsample=True: `F.interpolate(scale_factor=2)` of an UpsampleBlock is NOT written out; the
    convolution that consumes it (and its weight-gradient kernel) interpolates the (H/2, W/2)
    tensor while staging its input tile (descriptor code `pool = 2 / 3`).  Four dependent loads +
    the interpolation per staged element in the register-staged loaders can cost more than the
    `upsample_fwd` pass they replace, and the layer loses its TMA-staged path, so the default is
    False."""
    if upsample is not None:
        _MATH["fuse_up"] = bool(upsample)


def set_math(mode: str = "tf32x3", wgrad_tc: Optional[bool] = None,
             wgrad_math: Optional[str] = "auto") -> None:
    """Arithmetic of the convolution family:
      'tf32'   wgmma tensor cores, operands RN-rounded to TF32 (what stock PyTorch/cuDNN does by
               default on CUDA); ~1e-3 relative on the logits of a 17-layer Unet;
      'tf32x3' the same kernels with every operand split into a TF32 high and low part (three MMAs
               per product, fp32 accumulate): matches the reference's fp32 CPU results to ~1e-6;
      'fp32'   exact FFMA (CUDA-core) kernels.
    wgrad_math ('auto' | 'same' | 'tf32' | 'tf32x3'): arithmetic of the weight-gradient contraction
    only.  Its reduction runs over every pixel of the batch (K = N*H*W ~ 10^4..10^7 terms), so the
    unbiased RN operand rounding of single TF32 averages out there (relative error ~2^-12/sqrt(K)
    per term) instead of accumulating as in the K = 9*Cin forward / dgrad contractions, whose
    errors BatchNorm's backward then amplifies.  'auto' (default) therefore runs the weight
    gradients of 'tf32x3' in single TF32: measured on the 17-layer Unet against the exact-fp32
    mode, total gradient error 7.7e-4 (4x256^2) / 1.9e-4 (2x64^2) vs 7.6e-4 / 4e-6 with split
    weight gradients ('same') — tools/debug_wgrad_mix.py, tests/test_unet_gpu.py."""
    assert mode in _MODES, f"math mode must be one of {sorted(_MODES)}"
    _MATH["mode"] = _MODES[mode]
    assert wgrad_math in (None, "auto", "same", "tf32", "tf32x3")
    if wgrad_math == "auto":
        wgrad_math = "tf32" if mode == "tf32x3" else "same"
    _MATH["wgrad"] = None if wgrad_math in (None, "same") or mode == "fp32" else _MODES[wgrad_math]
    if wgrad_tc is not None:
        _MATH["wgrad_tc"] = bool(wgrad_tc)


def get_math() -> str:
    inv = {v: k for k, v in _MODES.items()}
    m = inv[_MATH["mode"]]
    if _MATH["wgrad"] is not None and _MATH["wgrad"] != _MATH["mode"]:
        m += "+wgrad-" + inv[_MATH["wgrad"]]
    return m


class Act:
    """Activation handle: NHWC tensor + pending affine + pending pool / 2x upsampling (see module
    docstring)."""
    __slots__ = ("t", "scale", "shift", "pool", "up", "parent", "grad", "grad_owned", "extra",
                 "needs_grad", "prod", "bn_sums")

    def __init__(self, t, scale=None, shift=None, pool=False, parent=None, needs_grad=True, up=None):
        self.t, self.scale, self.shift, self.pool = t, scale, shift, pool
        self.up = up                  # None | 'bilinear' | 'nearest': pending 2x upsampling
        self.parent = parent          # set for lazy pooled / upsampled views: gradients go to the parent
        self.grad = None              # d loss / d (affine(a)), full resolution of t
        self.grad_owned = False       # True: grad buffer is exclusively ours (in-place add ok)
        self.extra = None             # DilatedBlock direct taps (d loss / d a and d pre)
        self.needs_grad = needs_grad
        self.prod = None              # (mean, invstd) of the BatchNorm this tensor feeds — NOT the
                                      # record itself: Act <-> record cycles would keep every
                                      # activation alive until the cyclic GC runs
        self.bn_sums = None           # BatchNorm-backward sums of `grad`, when the kernel that
                                      # finished `grad` computed them on the way (pool backward)

    @property
    def shape(self):                  # logical NHWC shape seen by a consumer
        n, h, w, c = self.t.shape
        if self.up:
            return (n, 2 * h, 2 * w, c)
        return (n, h // 2, w // 2, c) if self.pool else (n, h, w, c)

    @property
    def C(self):
        return self.t.shape[3]

    def source(self) -> Source:
        code = ops.SRC_POOL if self.pool else (
            0 if not self.up else (ops.SRC_UP_BILINEAR if self.up == "bilinear" else ops.SRC_UP_NEAREST))
        return Source(self.t, self.scale, self.shift, code)

    def pending(self) -> bool:
        return bool(self.pool) or self.up is not None or self.scale is not None


def _acc_grad(act: Act, g: torch.Tensor, owned: bool) -> None:
    """act.grad (+)= g.  g may be a channel-slice view; `owned` says whether the caller hands over
    exclusive ownership of g's memory.  A buffer that is not exclusively ours (e.g. the gradient of
    a DilatedBlock sum shared by all its layers) is never written in place."""
    act.bn_sums = None                # any further contribution invalidates fused statistics
    if act.grad is None:
        act.grad, act.grad_owned = g, owned
        return
    if not act.grad_owned:
        own = torch.empty(act.grad.shape, device=g.device, dtype=torch.float32)
        ops.add_slice(act.grad, own, False)
        act.grad, act.grad_owned = own, True
    ops.add_slice(g, act.grad, True)


def _dense(g: torch.Tensor) -> torch.Tensor:
    """Contiguous NHWC copy of a channel-slice view (kernels that need ld == C)."""
    if g.is_contiguous():
        return g
    own = torch.empty(g.shape, device=g.device, dtype=torch.float32)
    ops.add_slice(g, own, False)
    return own


class _ConvRec:
    __slots__ = ("srcs", "out", "conv", "bn", "ks", "dil", "act", "slope", "math", "mean",
                 "invstd", "scale", "count", "needs_in_grad", "drop")


class _PointwiseAdapter:
    """Presents an nn.Linear as the 1x1 convolution it is when applied per pixel."""
    __slots__ = ("weight", "bias", "dilation", "stride", "padding", "_w4")

    def __init__(self, lin):
        self.weight, self.bias = lin.weight, lin.bias
        self.dilation, self.stride, self.padding = (1, 1), (1, 1), (0, 0)


class Tape:
    def __init__(self, training: bool, record: bool, comm=None):
        self.training = training      # BatchNorm uses batch statistics
        self.record = record          # keep what backward needs
        self.comm = comm              # optional: object with allreduce_sum_(tensor) for SyncBN
        self.ops = []                 # recorded (kind, payload) in forward order
        self.param_grads = {}         # nn.Parameter -> grad tensor
        self.alias = {}               # id(padded weight view) -> fn(grad) -> (nn.Parameter, grad)
        self.widths = []              # feature-map widths seen (get_downsample_factor)

    # ------------------------------------------------------------------ helpers
    def input(self, x_nhwc: torch.Tensor, needs_grad: bool = False) -> Act:
        return Act(x_nhwc, needs_grad=needs_grad)

    def _math_for(self, srcs: Sequence[Act], cout: int) -> int:
        if _MATH["mode"] != MATH_FP32 and ops.tc_supported([s.source() for s in srcs], cout):
            return _MATH["mode"]
        return MATH_FP32

    def _add_pgrad(self, p, g: torch.Tensor) -> None:
        if p is None:
            return
        h = self.alias.get(id(p))
        if h is not None:             # gradient of a padded / blocked copy of a parameter
            p, g = h(g)
            if p is None:
                return
        g = g.reshape(p.shape)
        if p in self.param_grads:
            self.param_grads[p] = self.param_grads[p] + g
        else:
            self.param_grads[p] = g

    # ------------------------------------------------------------------ convolution layer
    def conv(self, srcs: Union[Act, Sequence[Act]], conv_mod, bn_mod=None, slope: float = 1.0,
             act: int = ACT_LRELU, out_nchw: bool = False, out_t: Optional[torch.Tensor] = None,
             p_drop: float = 0.0) -> Act:
        """conv (+bias) -> activation -> [BatchNorm as a pending affine].
        conv_mod: nn.Conv2d / nn.Conv1d (k in {1,3}, stride 1, padding = dilation*(k//2));
        bn_mod: nn.BatchNorm2d/1d or None.  Reference: atomai/nets/blocks.py:61-76, 302-319."""
        if isinstance(srcs, Act):
            srcs = [srcs]
        srcs = list(srcs)
        n, h, w, _ = srcs[0].shape
        wt = conv_mod.weight
        cout = wt.shape[0]
        if wt.dim() == 4:
            ks = (wt.shape[2], wt.shape[3])
            dil = conv_mod.dilation[0]
        elif wt.dim() == 3:            # Conv1d: signals are (N, 1, L, C)
            ks = (1, wt.shape[2])
            dil = conv_mod.dilation[0]
        else:                          # nn.Linear applied per pixel == 1x1 convolution
            ks, dil = (1, 1), 1
        _check_conv(conv_mod, ks, dil)
        ctot = sum(s.C for s in srcs)
        assert ctot == wt.shape[1], f"conv expects {wt.shape[1]} input channels, got {ctot}"
        math = self._math_for(srcs, cout)
        d = ops.conv_desc([s.source() for s in srcs], n, h, w, cout, ks, dil, slope, math,
                          out_nchw, act)
        wp = ops.prep_weights(_w4(wt), ops.WMODE_FWD, math)
        dev = wt.device
        if out_t is not None:          # caller-provided (channel slice of a wider) output buffer
            assert not out_nchw and tuple(out_t.shape) == (n, h, w, cout)
        elif out_nchw:
            out_t = torch.empty((n, cout, h, w), device=dev, dtype=torch.float32)
        else:
            out_t = torch.empty((n, h, w, cout), device=dev, dtype=torch.float32)
        use_batch_stats = bn_mod is not None and (self.training or bn_mod.running_mean is None)
        stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64) if use_batch_stats else None
        bias = conv_mod.bias
        # nn.Dropout sits between the convolution and the LeakyReLU (blocks.py:68-70); inverted
        # dropout scales by 1/(1-p) > 0 or zeroes, so it commutes with the fused LeakyReLU and is
        # applied to the kernel's output, with the BatchNorm statistics taken after it.
        drop = None
        if p_drop > 0 and self.training:
            assert not out_nchw and act == ACT_LRELU
            drop = (float(p_drop), int(torch.randint(0, 2 ** 62, (1,)).item()))
        ops.conv_fwd(d, wp, None if bias is None else bias.detach(), out_t,
                     None if drop is not None else stats)
        if drop is not None:
            ops.dropout_(out_t, drop[0], drop[1], stats)
        self.widths.append(w)
        scale = shift = mean = invstd = None
        count = n * h * w
        if bn_mod is not None:
            assert not out_nchw
            scale = torch.empty(cout, device=dev, dtype=torch.float32)
            shift = torch.empty(cout, device=dev, dtype=torch.float32)
            if use_batch_stats:
                mean = torch.empty(cout, device=dev, dtype=torch.float32)
                invstd = torch.empty(cout, device=dev, dtype=torch.float32)
                mom = bn_mod.momentum if bn_mod.momentum is not None else 0.1
                fused = False
                if self.comm is not None:
                    count = self.comm.allreduce_count(count)
                    # one kernel: exchange of the statistics over NVLink peer memory + finalise
                    fused = getattr(self.comm, "bn_finalize_fused", lambda *a: False)(
                        stats, count, _d(bn_mod.weight), _d(bn_mod.bias), bn_mod.running_mean,
                        bn_mod.running_var, mom, bn_mod.eps, scale, shift, mean, invstd)
                    if not fused:
                        self.comm.allreduce_sum_(stats)
                if not fused:
                    ops.bn_finalize(stats, count, _d(bn_mod.weight), _d(bn_mod.bias),
                                    bn_mod.running_mean, bn_mod.running_var, mom, bn_mod.eps, True,
                                    scale, shift, mean, invstd)
                if bn_mod.num_batches_tracked is not None:
                    bn_mod.num_batches_tracked.add_(1)
            else:
                ops.bn_finalize(None, count, _d(bn_mod.weight), _d(bn_mod.bias),
                                bn_mod.running_mean, bn_mod.running_var, 0.0, bn_mod.eps, False,
                                scale, shift, None, None)
        out = Act(out_t, scale, shift)
        if self.record:
            r = _ConvRec()
            r.srcs, r.out, r.conv, r.bn, r.ks, r.dil = srcs, out, conv_mod, bn_mod, ks, dil
            r.act, r.slope, r.math, r.mean, r.invstd, r.scale, r.count = \
                act, slope, math, mean, invstd, scale, count
            r.needs_in_grad = any(s.needs_grad for s in srcs)
            r.drop = drop
            if bn_mod is not None and mean is not None:
                out.prod = (mean, invstd)
            assert not (bn_mod is not None and not use_batch_stats), \
                "backward through eval-mode BatchNorm is not supported"
            assert not out_nchw or True
            self.ops.append(("conv", r))
        return out

    def _conv_bwd(self, r: _ConvRec) -> None:
        out = r.out
        a = out.t
        if a.dim() == 4 and a.shape[-1] != r.conv.weight.shape[0]:
            # NCHW output (flatten -> Linear consumers): gradient arrives NCHW; bring to NHWC
            raise NotImplementedError("backward through an NCHW-stored conv output")
        dy = out.grad
        n, h, w, cout = a.shape
        dev = a.device
        sums = None
        if r.bn is not None:
            assert dy is not None, "BatchNorm output has no gradient"
            sums = out.bn_sums
            out.bn_sums = None
            if sums is None:
                sums = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
                ops.bn_bwd_reduce(dy, a, r.mean, r.invstd, sums)
            # gamma/beta gradients come from the LOCAL sums (the gradient bucket sums them over
            # ranks like every other parameter, as torch's SyncBatchNorm does); only the dx
            # formula needs the global sums.
            self._add_pgrad(r.bn.bias, sums[:cout].float())
            self._add_pgrad(r.bn.weight, sums[cout:].float())
            if self.comm is not None:
                self.comm.allreduce_sum_(sums)
        dpre = torch.empty((n, h, w, cout), device=dev, dtype=torch.float32)
        dbias = torch.zeros(cout, device=dev, dtype=torch.float64) if r.conv.bias is not None else None
        ops.bn_act_bwd(dy, a, r.mean, r.invstd, r.scale if r.bn is not None else None, sums,
                       r.count, out.extra, r.act, r.slope, dpre, None if r.drop else dbias)
        if r.drop:            # same (seed, index) mask on the gradient; bias gradient after it
            dsum = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
            ops.dropout_(dpre, r.drop[0], r.drop[1], dsum)
            if dbias is not None:
                dbias = dsum[:cout]
        out.grad = None
        out.extra = None
        if dbias is not None:
            self._add_pgrad(r.conv.bias, dbias.float())
        # weight gradient
        wt = r.conv.weight
        srcs_s = [s.source() for s in r.srcs]
        dw = torch.zeros((wt.shape[0], wt.shape[1], r.ks[0], r.ks[1]), device=dev,
                         dtype=torch.float32)
        wmath = r.math if (r.math == MATH_FP32 or _MATH["wgrad"] is None) else _MATH["wgrad"]
        dsc = ops.conv_desc(srcs_s, n, h, w, cout, r.ks, r.dil, 1.0, wmath)
        if wmath != MATH_FP32 and not (_MATH["wgrad_tc"] and ops.conv_supported(dsc, 1)):
            dsc.math = MATH_FP32
        ops.conv_wgrad(dsc, dpre, dw)
        self._add_pgrad(wt, dw)
        # data gradient
        if r.needs_in_grad:
            ctot = wt.shape[1]
            dsrc = [Source(dpre)]
            dmath = _MATH["mode"] if (_MATH["mode"] != MATH_FP32 and ops.tc_supported(dsrc, ctot)) \
                else MATH_FP32
            wpd = ops.prep_weights(_w4(wt), ops.WMODE_DGRAD, dmath)
            dd = ops.conv_desc(dsrc, n, h, w, ctot, r.ks, r.dil, 1.0, dmath)
            dx = torch.empty((n, h, w, ctot), device=dev, dtype=torch.float32)
            ops.conv_fwd(dd, wpd, None, dx, None)
            c0 = 0
            for s in r.srcs:
                view = dx[..., c0:c0 + s.C] if len(r.srcs) > 1 else dx
                c0 += s.C
                if not s.needs_grad:
                    continue
                if s.pool:
                    self._pool_grad(s.parent, view)
                elif s.up:
                    self._up_grad(s, view)
                else:
                    _acc_grad(s, view, True)

    @staticmethod
    def _pool_grad(tgt: Act, gp: torch.Tensor) -> None:
        """tgt.grad (+)= unpool(gp): scatter to the arg-max positions of tgt's affine'd windows."""
        acc = tgt.grad is not None
        if not acc:
            tgt.grad = torch.empty(tgt.t.shape, device=gp.device, dtype=torch.float32)
            tgt.grad_owned = True
        elif not tgt.grad_owned:      # (an owned channel-slice view is accumulated into in place)
            own = torch.empty(tgt.t.shape, device=gp.device, dtype=torch.float32)
            ops.add_slice(tgt.grad, own, False)
            tgt.grad, tgt.grad_owned = own, True
        # The pooled consumer is normally the LAST one to deliver its gradient (it runs first in
        # forward, so last in backward): let the scatter kernel also produce the BatchNorm-backward
        # sums of the finished gradient; _acc_grad drops them again if something else follows.
        sums = None
        if tgt.prod is not None and ops.pool_bwd_stats_ok(tgt.C) and not _NO_POOLSTATS:
            mean, invstd = tgt.prod
            sums = torch.zeros(2 * tgt.C, device=gp.device, dtype=torch.float64)
            ops.pool_bwd(gp, tgt.t, tgt.scale, tgt.shift, tgt.grad, acc, mean, invstd, sums)
        else:
            ops.pool_bwd(gp, tgt.t, tgt.scale, tgt.shift, tgt.grad, acc)
        tgt.bn_sums = sums

    # ------------------------------------------------------------------ pooling / upsampling
    def pool(self, x: Act) -> Act:
        """F.max_pool2d(x, 2, 2) as a pending transform (atomai/nets/fcnn.py:123-127)."""
        if x.pool or x.up:
            x = self.materialize(x)
        assert x.t.shape[1] % 2 == 0 and x.t.shape[2] % 2 == 0, \
            "2x2 max-pool needs even spatial dimensions"
        return Act(x.t, x.scale, x.shift, pool=True, parent=x, needs_grad=x.needs_grad)

    def upsample(self, x: Act, mode: str = "bilinear") -> Act:
        """F.interpolate(scale_factor=2, mode) (atomai/nets/blocks.py:130-131) as a PENDING
        transform: the consuming convolution interpolates while it stages its input tile
        (forward, dgrad's source routing and the weight gradient), so the 4x larger tensor is
        never written.  Other consumers materialise it (`materialize`)."""
        if x.pool or x.up:
            x = self.materialize(x)
        assert mode in ("bilinear", "nearest")
        if not _MATH["fuse_up"]:
            return self.materialize(Act(x.t, x.scale, x.shift, parent=x, needs_grad=x.needs_grad, up=mode))
        return Act(x.t, x.scale, x.shift, parent=x, needs_grad=x.needs_grad, up=mode)

    @staticmethod
    def _up_grad(s: Act, g: torch.Tensor) -> None:
        """parent.grad (+)= upsample^T(g) (g: gradient w.r.t. the upsampled, affine'd values)."""
        x = s.parent
        if not x.needs_grad:
            return
        dx = torch.empty(x.t.shape, device=g.device, dtype=torch.float32)
        ops.upsample_bwd(g, dx, s.up == "bilinear")
        _acc_grad(x, dx, True)

    def materialize(self, x: Act, nchw: bool = False) -> Act:
        """Apply the pending affine / pool and write the result (module boundaries only)."""
        if not x.pending() and not nchw:
            return x
        n, h, w, c = x.shape
        dev = x.t.device
        if x.up:
            assert not nchw
            src = x.t
            if x.scale is not None:       # affine and interpolation commute (weights sum to one)
                src = torch.empty(x.t.shape, device=dev, dtype=torch.float32)
                ops.affine(x.t, x.scale, x.shift, src)
            out_t = torch.empty((n, h, w, c), device=dev, dtype=torch.float32)
            ops.upsample_fwd(src, out_t, x.up == "bilinear")
        elif x.pool:
            assert not nchw
            out_t = torch.empty((n, h, w, c), device=dev, dtype=torch.float32)
            ops.pool_fwd(x.t, x.scale, x.shift, out_t)
        elif nchw:
            out_t = torch.empty((n, c, h, w), device=dev, dtype=torch.float32)
            ops.affine(x.t, x.scale, x.shift, out_t, out_nchw=True)
        else:
            out_t = torch.empty((n, h, w, c), device=dev, dtype=torch.float32)
            ops.affine(x.t, x.scale, x.shift, out_t)
        out = Act(out_t, needs_grad=x.needs_grad)
        if self.record:
            self.ops.append(("mat", (x, out, nchw)))
        return out

    def _mat_bwd(self, rec) -> None:
        x, out, nchw = rec
        if not x.needs_grad or out.grad is None:
            return
        g = out.grad
        if nchw:                       # gradient arrives as (N,C,H,W); view it as NHWC
            g = g.permute(0, 2, 3, 1)
            if not (g.stride(3) == 1):
                g = g.contiguous()
        owned = out.grad_owned
        out.grad = None
        if x.pool:
            self._pool_grad(x.parent, g)
        elif x.up:
            self._up_grad(x, g)
        else:
            _acc_grad(x, g, owned)

    # ------------------------------------------------------------------ DilatedBlock sum
    def dilated_sum(self, layers: List[Act], slope: float) -> Act:
        """sum over layers of (conv out + LeakyReLU out + [BN out]) — blocks.py:321-329."""
        n, h, w, c = layers[0].t.shape
        out_t = torch.empty((n, h, w, c), device=layers[0].t.device, dtype=torch.float32)
        ops.dilated_sum([l.t for l in layers], [l.scale for l in layers],
                        [l.shift for l in layers], slope, out_t)
        out = Act(out_t)
        if self.record:
            self.ops.append(("dsum", (layers, out)))
        return out

    def _dsum_bwd(self, rec) -> None:
        layers, out = rec
        g = out.grad
        if g is None:
            return
        g = _dense(g)
        out.grad = None
        for l in layers:
            l.extra = g                # direct taps on a_l and pre_l (read-only, shared)
            if l.scale is not None:    # BN output also enters the sum
                _acc_grad(l, g, False)


    def add(self, a: Act, b: Act) -> Act:
        """a + b (rDecoderNet's skip connections, atomai/nets/ed.py:632-637)."""
        if a.pending():
            a = self.materialize(a)
        if b.pending():
            b = self.materialize(b)
        out_t = torch.empty(a.t.shape, device=a.t.device, dtype=torch.float32)
        ops.add_slice(a.t, out_t, False)
        ops.add_slice(b.t, out_t, True)
        out = Act(out_t)
        if self.record:
            self.ops.append(("custom", _AddRec(a, b, out)))
        return out

    def cat(self, xs: Sequence[Act]) -> Act:
        """torch.cat(xs, 1) written out (pending affines applied on the way) — for concatenations a
        convolution cannot take as separate sources (more than two, or channel counts that are not
        multiples of 4: ResHedNet's side outputs, atomai/nets/fcnn.py:295)."""
        xs = [self.materialize(x) if x.pool else x for x in xs]
        n, h, w, _ = xs[0].t.shape
        ctot = sum(x.C for x in xs)
        out_t = torch.empty((n, h, w, ctot), device=xs[0].t.device, dtype=torch.float32)
        c0, parts = 0, []
        for x in xs:
            sl = out_t[..., c0:c0 + x.C]
            if x.scale is not None:
                ops.affine(x.t, x.scale, x.shift, sl)
            else:
                ops.add_slice(x.t, sl, False)
            parts.append((x, c0, c0 + x.C))
            c0 += x.C
        out = Act(out_t)
        if self.record:
            self.ops.append(("custom", _CatRec(out, parts)))
        return out

    def bn_res_act(self, x: Act, res: Optional[Act], slope: float) -> Act:
        """LeakyReLU(BatchNorm(x) [+ res]) — the tail of a ResBlock (atomai/nets/blocks.py:205-213:
        `out = bn(out); out += residual; out = leaky_relu(out)`) as one pass: x carries the
        BatchNorm as its pending affine."""
        assert not x.pool and slope > 0
        if res is not None and res.pending():
            res = self.materialize(res)
        out_t = torch.empty(x.t.shape, device=x.t.device, dtype=torch.float32)
        ops.affine_res_act(x.t, x.scale, x.shift, None if res is None else res.t, slope, out_t)
        out = Act(out_t)
        if self.record:
            self.ops.append(("custom", _ResActRec(x, res, out, slope)))
        return out

    def resize(self, x: Act, factor: int, mode: str = "bilinear") -> Act:
        """F.interpolate(x, size=factor*(h, w), mode) (atomai/nets/fcnn.py:292-293)."""
        if factor == 1:
            return x
        if x.pending():
            x = self.materialize(x)
        n, h, w, c = x.t.shape
        out_t = torch.empty((n, factor * h, factor * w, c), device=x.t.device, dtype=torch.float32)
        ops.resize_fwd(x.t, out_t, factor, mode == "bilinear")
        out = Act(out_t, needs_grad=x.needs_grad)
        if self.record:
            self.ops.append(("custom", _ResizeRec(x, out, factor, mode == "bilinear")))
        return out

    # ------------------------------------------------------------------ dense layers
    def pointwise(self, x: Act, lin_mod, slope: float = 1.0, act: int = ACT_LRELU) -> Act:
        """nn.Linear applied to every pixel's channel vector (rDecoderNet's fc_decoder / out,
        atomai/nets/ed.py:620-624,639) = 1x1 convolution on the tensor cores."""
        return self.conv(x, _PointwiseAdapter(lin_mod), None, slope, act)

    def linear(self, x: Act, lin_mod, act: Optional[int] = None) -> Act:
        """nn.Linear on a (B, K) activation stored as (B,1,1,K) — the skinny heads of the VAE /
        ImSpec nets (atomai/nets/ed.py:64,273-274,503-505) and the DKL MLP (nets/gp.py:23-26).
        act: None (identity), ACT_TANH, or 'relu'."""
        if x.pending():
            x = self.materialize(x)
        b, k = x.t.shape[0], x.t.shape[3]
        assert x.t.shape[1] == 1 and x.t.shape[2] == 1 and x.t.is_contiguous()
        w, bias = lin_mod.weight.detach(), _d(lin_mod.bias)
        o = w.shape[0]
        y = torch.empty((b, 1, 1, o), device=w.device, dtype=torch.float32)
        if act is None:
            ops.linear_fwd(x.t.view(b, k), w, bias, y.view(b, o))
        else:
            a_id, slope = (ACT_TANH, 1.0) if act == ACT_TANH else (ACT_LRELU, 0.0)
            ops.gemm(x.t, k, 1, w, 1, k, y, o, b, o, k, bias, a_id, slope)
        out = Act(y, needs_grad=True)
        if self.record:
            self.ops.append(("lin", (x, out, lin_mod, act)))
        return out

    def mlp(self, x: Act, lins: Sequence, acts: Sequence) -> Act:
        """Chain of nn.Linear (+ReLU / tanh) layers on a (B,1,1,K) activation — the DKL feature
        extractor (atomai/nets/gp.py:14-26: feat -> 1000 -> 500 -> 50 -> embedim) — on the wgmma
        convolution kernel: the B rows become the pixels of a (1, B/8, 8, K) image, each layer is a
        1x1 convolution with fused bias + activation, wide layers run as column blocks of <= 256
        outputs writing channel slices of one buffer.  Channel counts are zero-padded to the MMA
        granularity (K % 8, N % 16) once per call; padded rows / channels stay exact zeros through
        forward and backward.  fp32 math mode and tiny batches take the per-layer SIMT path."""
        if x.pending():
            x = self.materialize(x)
        b, k = x.t.shape[0], x.t.shape[3]
        if _MATH["mode"] == MATH_FP32 or b < 64:
            for lin, a in zip(lins, acts):
                x = self.linear(x, lin, a)
            return x
        dev = x.t.device
        rows, kp = -(-b // 8) * 8, -(-k // 8) * 8
        if rows != b or kp != k:
            xin = torch.zeros((1, rows // 8, 8, kp), device=dev, dtype=torch.float32)
            xin.view(rows, kp)[:b, :k] = x.t.view(b, k)
        else:
            xin = x.t.view(1, rows // 8, 8, k)
        cur = Act(xin, needs_grad=x.needs_grad)
        if self.record:
            self.ops.append(("custom", _PadRec(x, cur, b, k)))
        for lin, a in zip(lins, acts):
            o, kk = lin.weight.shape
            op = -(-o // 16) * 16
            kcur = cur.t.shape[3]
            wpad = torch.zeros((op, kcur), device=dev, dtype=torch.float32)
            wpad[:o, :kk] = lin.weight.detach()
            bpad = torch.zeros(op, device=dev, dtype=torch.float32)
            if lin.bias is not None:
                bpad[:o] = lin.bias.detach()
            nblk = -(-op // 256)
            per = -(-(op // 16) // nblk) * 16
            buf = torch.empty((1, rows // 8, 8, op), device=dev, dtype=torch.float32)
            a_id, slope = (ACT_TANH, 1.0) if a == ACT_TANH else \
                (ACT_LRELU, 0.0 if a == "relu" else 1.0)
            blocks = []
            for c0 in range(0, op, per):
                c1 = min(op, c0 + per)
                ad = _PaddedBlock(wpad[c0:c1], bpad[c0:c1])
                self.alias[id(ad.weight)] = _unpad_w(lin.weight, c0, min(c1, o), kk)
                self.alias[id(ad.bias)] = _unpad_b(lin.bias, c0, min(c1, o))
                blk = self.conv(cur, ad, None, slope, a_id, out_t=buf[..., c0:c1])
                blocks.append((blk, c0, c1))
            cur = Act(buf)
            if self.record:
                self.ops.append(("custom", _SplitRec(cur, blocks)))
        o_last = lins[-1].weight.shape[0]
        y = torch.empty((b, 1, 1, o_last), device=dev, dtype=torch.float32)
        y.view(b, o_last).copy_(cur.t.view(rows, -1)[:b, :o_last])
        out = Act(y)
        if self.record:
            self.ops.append(("custom", _PadRec(cur, out, b, o_last, unpad=True)))
        return out

    def _lin_bwd(self, rec) -> None:
        x, out, lin_mod, act = rec
        if out.grad is None:
            return
        dy = _dense(out.grad)
        out.grad = None
        b, k, o = x.t.shape[0], x.t.shape[3], out.t.shape[3]
        if act is not None:
            a_id, slope = (ACT_TANH, 1.0) if act == ACT_TANH else (ACT_LRELU, 0.0)
            dpre = torch.empty_like(out.t)
            ops.bn_act_bwd(dy, out.t, None, None, None, None, 1.0, None, a_id, slope, dpre, None)
            dy = dpre
        w = lin_mod.weight.detach()
        dx = torch.empty_like(x.t) if x.needs_grad else None
        dw = torch.empty_like(w)
        db = torch.empty(o, device=w.device, dtype=torch.float32) if lin_mod.bias is not None else None
        ops.linear_bwd(x.t.view(b, k), w, dy.view(b, o), None if dx is None else dx.view(b, k), dw, db)
        self._add_pgrad(lin_mod.weight, dw)
        if db is not None:
            self._add_pgrad(lin_mod.bias, db)
        if dx is not None:
            _acc_grad(x, dx, True)

    def flatten(self, x: Act) -> Act:
        """(N,H,W,C) -> (N,1,1,C*H*W) in the reference's NCHW order (`x.reshape(-1, C*H*W)`)."""
        x = self.materialize(x)
        n, h, w, c = x.t.shape
        y = torch.empty((n, 1, 1, c * h * w), device=x.t.device, dtype=torch.float32)
        if c == 1 or h * w == 1:
            y.copy_(x.t.reshape(n, 1, 1, -1))
        else:
            ops.transpose(x.t, y, n, h * w, c)
        out = Act(y, needs_grad=x.needs_grad)
        if self.record:
            self.ops.append(("flat", (x, out, True)))
        return out

    def unflatten(self, x: Act, c: int, h: int, w: int) -> Act:
        """(N,1,1,C*H*W) in NCHW order -> (N,H,W,C)."""
        x = self.materialize(x)
        n = x.t.shape[0]
        y = torch.empty((n, h, w, c), device=x.t.device, dtype=torch.float32)
        if c == 1 or h * w == 1:
            y.copy_(x.t.reshape(n, h, w, c))
        else:
            ops.transpose(x.t.contiguous(), y, n, c, h * w)
        out = Act(y, needs_grad=x.needs_grad)
        if self.record:
            self.ops.append(("flat", (x, out, False)))
        return out

    def _flat_bwd(self, rec) -> None:
        x, out, fwd_is_flatten = rec
        if out.grad is None or not x.needs_grad:
            return
        g = _dense(out.grad)
        out.grad = None
        gx = torch.empty_like(x.t)
        if fwd_is_flatten:
            n, h, w, c = x.t.shape
            if c == 1 or h * w == 1:
                gx.copy_(g.reshape(x.t.shape))
            else:
                ops.transpose(g, gx, n, c, h * w)
        else:
            n, h, w, c = out.t.shape
            if c == 1 or h * w == 1:
                gx.copy_(g.reshape(x.t.shape))
            else:
                ops.transpose(g, gx, n, h * w, c)
        _acc_grad(x, gx, True)

    def coord_latent(self, mod, hw, z: Act, phi: Optional[Act], dx: Optional[Act],
                     tanh_act: bool) -> Act:
        """coord_latent + transform_coordinates fused (atomai/nets/ed.py:672-687,
        atomai/utils/coords.py:57-83): h0[b, p, :] = act(Wc (R(phi_b) g_p + dx_b) + bc + Wz z_b)."""
        h, w = hw
        b = z.t.shape[0]
        zt = z.t.reshape(b, -1).contiguous()
        wc, bc = mod.fc_coord.weight.detach(), _d(mod.fc_coord.bias)
        wz = mod.fc_latent.weight.detach()
        hid = wc.shape[0]
        ph = None if phi is None else phi.t.reshape(b).contiguous()
        dxt = None if dx is None else dx.t.reshape(b, 2).contiguous()
        d = ops.coord_latent_desc(b, h, w, zt, ph, dxt, wc, bc, wz, tanh_act)
        h0 = torch.empty((b, h, w, hid), device=wc.device, dtype=torch.float32)
        ops.coord_latent_fwd(d, h0)
        out = Act(h0)
        if self.record:
            self.ops.append(("cl", (mod, (h, w), z, phi, dx, tanh_act, zt, ph, dxt, out)))
        return out

    def _cl_bwd(self, rec) -> None:
        mod, (h, w), z, phi, dx, tanh_act, zt, ph, dxt, out = rec
        if out.grad is None:
            return
        g = _dense(out.grad)
        out.grad = None
        b, hid = zt.shape[0], out.t.shape[3]
        dev = g.device
        if tanh_act:
            dpre = torch.empty_like(out.t)
            ops.bn_act_bwd(g, out.t, None, None, None, None, 1.0, None, ACT_TANH, 1.0, dpre, None)
            g = dpre
        wc, bc = mod.fc_coord.weight.detach(), _d(mod.fc_coord.bias)
        wz = mod.fc_latent.weight.detach()
        dwc = torch.zeros_like(wc)
        dbc = torch.zeros(hid, device=dev, dtype=torch.float32)
        sb = torch.zeros((b, hid), device=dev, dtype=torch.float32)
        dphi = torch.zeros(b, device=dev, dtype=torch.float32) if phi is not None else None
        ddx = torch.zeros((b, 2), device=dev, dtype=torch.float32) if dx is not None else None
        d = ops.coord_latent_desc(b, h, w, zt, ph, dxt, wc, bc, wz, tanh_act)
        ops.coord_latent_bwd(d, g, dwc, dbc, sb, dphi, ddx)
        self._add_pgrad(mod.fc_coord.weight, dwc)
        if mod.fc_coord.bias is not None:
            self._add_pgrad(mod.fc_coord.bias, dbc)
        zd = zt.shape[1]
        dwz = torch.empty_like(wz)                       # dWz[h][k] = sum_b sb[b][h] z[b][k]
        ops.gemm(sb, 1, hid, zt, zd, 1, dwz, zd, hid, zd, b)
        self._add_pgrad(mod.fc_latent.weight, dwz)
        if z.needs_grad:
            dz = torch.empty((b, 1, 1, zd), device=dev, dtype=torch.float32)
            ops.gemm(sb, hid, 1, wz, zd, 1, dz, zd, b, zd, hid)   # dz = sb @ Wz
            _acc_grad(z, dz, True)
        if phi is not None and phi.needs_grad:
            _acc_grad(phi, dphi.reshape(phi.t.shape), True)
        if dx is not None and dx.needs_grad:
            _acc_grad(dx, ddx.reshape(dx.t.shape), True)

    # ------------------------------------------------------------------ backward driver
    def backward_no_seed(self) -> None:
        self._replay()

    def backward(self, out: Act, grad_out_nhwc: torch.Tensor) -> None:
        out.grad, out.grad_owned = grad_out_nhwc, False
        self._replay()

    def _replay(self) -> None:
        for kind, rec in reversed(self.ops):
            if kind == "conv":
                self._conv_bwd(rec)
            elif kind == "mat":
                self._mat_bwd(rec)
            elif kind == "dsum":
                self._dsum_bwd(rec)
            elif kind == "lin":
                self._lin_bwd(rec)
            elif kind == "flat":
                self._flat_bwd(rec)
            elif kind == "cl":
                self._cl_bwd(rec)
            elif kind == "custom":
                rec.backward(self)
            else:
                raise RuntimeError(kind)
        self.ops = []


class _PaddedBlock:
    """A row block of a zero-padded nn.Linear weight, presented as a 1x1 convolution."""
    __slots__ = ("weight", "bias", "dilation", "stride", "padding")

    def __init__(self, w, b):
        self.weight, self.bias = w, b
        self.dilation, self.stride, self.padding = (1, 1), (1, 1), (0, 0)


def _unpad_w(param, r0, r1, k):
    def fn(g):
        if r1 <= r0:
            return None, None
        full = torch.zeros_like(param)
        full[r0:r1] = g.reshape(g.shape[0], -1)[:r1 - r0, :k]
        return param, full
    return fn


def _unpad_b(param, r0, r1):
    def fn(g):
        if param is None or r1 <= r0:
            return None, None
        full = torch.zeros_like(param)
        full[r0:r1] = g.reshape(-1)[:r1 - r0]
        return param, full
    return fn


class _AddRec:
    def __init__(self, a, b, out):
        self.a, self.b, self.out = a, b, out

    def backward(self, tape):
        g = self.out.grad
        self.out.grad = None
        if g is None:
            return
        g = _dense(g)
        for s_ in (self.a, self.b):
            if s_.needs_grad:
                _acc_grad(s_, g, False)


class _CatRec:
    def __init__(self, out, parts):
        self.out, self.parts = out, parts

    def backward(self, tape):
        g = self.out.grad
        self.out.grad = None
        if g is None:
            return
        for x, c0, c1 in self.parts:
            if x.needs_grad:
                _acc_grad(x, g[..., c0:c1], False)


class _ResActRec:
    def __init__(self, x, res, out, slope):
        self.x, self.res, self.out, self.slope = x, res, out, slope

    def backward(self, tape):
        dy = self.out.grad
        self.out.grad = None
        if dy is None:
            return
        g = torch.empty(self.out.t.shape, device=dy.device, dtype=torch.float32)
        ops.lrelu_mask_bwd(dy, self.out.t, self.slope, g)
        shared = self.res is not None and self.res.needs_grad
        if self.x.needs_grad:
            _acc_grad(self.x, g, not shared)
        if shared:
            _acc_grad(self.res, g, False)


class _ResizeRec:
    def __init__(self, x, out, factor, bilinear):
        self.x, self.out, self.factor, self.bilinear = x, out, factor, bilinear

    def backward(self, tape):
        g = self.out.grad
        self.out.grad = None
        if g is None or not self.x.needs_grad:
            return
        dx = torch.zeros(self.x.t.shape, device=g.device, dtype=torch.float32)
        ops.resize_bwd(_dense(g), dx, self.factor, self.bilinear)
        _acc_grad(self.x, dx, True)


class _PadRec:
    """(B,1,1,K) <-> zero-padded (1, rows/8, 8, Kp) copy at the two ends of Tape.mlp."""
    def __init__(self, src, dst, b, k, unpad=False):
        self.src, self.dst, self.b, self.k, self.unpad = src, dst, b, k, unpad

    def backward(self, tape):
        src, dst = self.src, self.dst
        if dst.grad is None or not src.needs_grad:
            dst.grad = None
            return
        g = _dense(dst.grad)
        dst.grad = None
        gs = torch.zeros_like(src.t)
        if self.unpad:      # forward sliced rows/channels out of the padded buffer
            gs.view(gs.shape[1] * gs.shape[2], -1)[:self.b, :self.k] = g.view(self.b, self.k)
        else:               # forward copied into the padded buffer
            gs.view(self.b, self.k).copy_(g.view(g.shape[1] * g.shape[2], -1)[:self.b, :self.k])
        _acc_grad(src, gs, True)


class _SplitRec:
    """Column blocks of one layer write channel slices of `merged`; route its gradient back."""
    def __init__(self, merged, blocks):
        self.merged, self.blocks = merged, blocks

    def backward(self, tape):
        g = self.merged.grad
        self.merged.grad = None
        if g is None:
            return
        for blk, c0, c1 in self.blocks:
            blk.grad, blk.grad_owned = g[..., c0:c1], False


def _d(p):
    return None if p is None else p.detach()


def _w4(w: torch.Tensor) -> torch.Tensor:
    """Weight as OIHW: Conv2d as is, Conv1d (O,I,k) -> (O,I,1,k), Linear (O,I) -> (O,I,1,1)."""
    w = w.detach()
    if w.dim() == 3:
        return w.unsqueeze(2)
    if w.dim() == 2:
        return w.reshape(w.shape[0], w.shape[1], 1, 1)
    return w


def _check_conv(m, ks, dil) -> None:
    k = ks[1]
    stride = m.stride[0] if isinstance(m.stride, tuple) else m.stride
    pad = m.padding[-1] if isinstance(m.padding, tuple) else m.padding
    if k not in (1, 3) or ks[0] not in (1, 3):
        raise NotImplementedError(f"native conv supports kernel sizes 1 and 3, got {ks}")
    if stride != 1:
        raise NotImplementedError("native conv supports stride 1 only")
    if pad != dil * (k // 2):
        raise NotImplementedError(f"native conv needs 'same' padding (padding={pad}, "
                                  f"dilation={dil}, kernel={k})")


# ---------------------------------------------------------------------- autograd boundary
class _NetFn(torch.autograd.Function):
    """One network call = one autograd node.  inputs: (module, comm, x, *params)."""

    @staticmethod
    def forward(ctx, module, comm, grad_on, x, *params):
        # (autograd disables grad mode inside forward, so the caller passes it in)
        record = grad_on and any(p.requires_grad for p in params)
        x_needs = grad_on and x.requires_grad
        tape = Tape(module.training, record or x_needs, comm)
        xin = _to_nhwc(x)
        a_in = tape.input(xin, needs_grad=x_needs)
        out = module._emit(tape, a_in)
        out = tape.materialize(out)
        ctx.tape, ctx.out, ctx.a_in, ctx.params = tape, out, a_in, params
        ctx.x_needs = x_needs
        ctx.nparams = len(params)
        res = out.t.permute(0, 3, 1, 2)
        if getattr(module, "_squeeze_h", False):
            res = res.squeeze(2)
        return res

    @staticmethod
    def backward(ctx, g):
        tape, out = ctx.tape, ctx.out
        if getattr(g, "dim", None) and g.dim() == 3:
            g = g.unsqueeze(2)
        g = g.permute(0, 2, 3, 1)
        if not g.is_contiguous():
            g = g.contiguous()
        tape.backward(out, g)
        grads = tuple(tape.param_grads.get(p) for p in ctx.params)
        gx = None
        if ctx.x_needs and ctx.a_in.grad is not None:
            gx = ctx.a_in.grad.permute(0, 3, 1, 2)
        tape.param_grads = {}
        return (None, None, None, gx) + grads


class _MultiFn(torch.autograd.Function):
    """General boundary: emit(tape, *acts) -> Act or tuple of Acts.  Inputs/outputs are NHWC-shaped
    tensors already ((B,1,1,K) for vectors); the caller reshapes at the API surface."""

    @staticmethod
    def forward(ctx, module, emit, comm, grad_on, n_in, *tensors):
        ins, params = tensors[:n_in], tensors[n_in:]
        in_needs = [grad_on and t.requires_grad for t in ins]
        record = grad_on and (any(p.requires_grad for p in params) or any(in_needs))
        tape = Tape(module.training, record, comm)
        acts = [tape.input(t.detach().contiguous(), needs_grad=nd) for t, nd in zip(ins, in_needs)]
        outs = emit(tape, *acts)
        single = isinstance(outs, Act)
        outs = [outs] if single else list(outs)
        outs = [tape.materialize(o) for o in outs]
        ctx.tape, ctx.outs, ctx.acts, ctx.params, ctx.in_needs = tape, outs, acts, params, in_needs
        res = tuple(o.t for o in outs)
        return res[0] if single else res

    @staticmethod
    def backward(ctx, *gs):
        tape = ctx.tape
        first = True
        for o, g in zip(ctx.outs, gs):
            if g is not None:
                o.grad, o.grad_owned = g.contiguous(), False
        # replay (Tape.backward expects one seeded output; seed all, then run the op loop)
        out0 = ctx.outs[0]
        seed = out0.grad
        tape.backward(out0, seed) if seed is not None else tape.backward_no_seed()
        grads_in = tuple(a.grad if nd else None for a, nd in zip(ctx.acts, ctx.in_needs))
        grads_in = tuple(None if g is None else _dense(g) for g in grads_in)
        grads_p = tuple(tape.param_grads.get(p) for p in ctx.params)
        tape.param_grads = {}
        return (None, None, None, None, None) + grads_in + grads_p


def run_multi(module, emit, inputs, comm=None):
    """Execute `emit(tape, *acts)` natively; `inputs` are NHWC-shaped CUDA tensors."""
    params = [p for p in module.parameters()]
    for t in inputs:
        if not t.is_cuda:
            raise RuntimeError("atomai_b200 networks run on CUDA (sm_90a) only; there is no CPU path")
    return _MultiFn.apply(module, emit, comm, torch.is_grad_enabled(), len(inputs), *inputs, *params)


def _to_nhwc(x: torch.Tensor) -> torch.Tensor:
    """(N,C,H,W) or (N,C,L) -> contiguous (N,H,W,C) without a copy when C == 1 or channels_last."""
    if x.dim() == 3:
        x = x.unsqueeze(2)
    assert x.dim() == 4, f"expected NCHW input, got shape {tuple(x.shape)}"
    if not x.is_cuda:
        raise RuntimeError("atomai_b200 networks run on CUDA (sm_90a) only; there is no CPU path")
    if x.dtype != torch.float32:
        x = x.float()
    xp = x.permute(0, 2, 3, 1)
    if not xp.is_contiguous():
        xp = xp.contiguous()
    return xp


def run(module, x: torch.Tensor, comm=None) -> torch.Tensor:
    """Execute `module` (anything with _emit(tape, Act) -> Act) natively on x."""
    params = [p for p in module.parameters()]
    return _NetFn.apply(module, comm if comm is not None else getattr(module, "_comm", None),
                        torch.is_grad_enabled(), x, *params)


def probe_downsample_factor(model, dims=(1, 64, 64)) -> float:
    """max/min feature-map width of a network (utils.nn.get_downsample_factor)."""
    p = next(model.parameters())
    x = torch.randn(1, *dims, device=p.device)
    was_training = model.training
    model.eval()
    tape = Tape(False, False)
    with torch.no_grad():
        model._emit(tape, tape.input(_to_nhwc(x)))
    model.train(was_training)
    return max(tape.widths) / min(tape.widths)
