"""
Loss functions for the native path.  `select_loss` has the reference's contract
(atomai/losses_metrics/losses.py:139-174): the returned criteria are nn.Modules whose names and
reprs match torch's (`str(criterion) == "CrossEntropyLoss()"`, test/trainers/test_trainer.py:59-74)
but whose forward/backward run as fused sm_90a kernels: one pass computes the summed loss, the
backward pass recomputes the softmax and writes d(logits) scaled by the upstream gradient read from
device memory (no host synchronisation).
"""
import torch

from .. import ops


def _nhwc_view(t: torch.Tensor) -> torch.Tensor:
    """(N,C,...) logits -> (N,H,W,C) view/copy with channels innermost."""
    if t.dim() == 2:                       # (N, C)
        return t.reshape(t.shape[0], 1, 1, t.shape[1]).contiguous()
    if t.dim() == 3:                       # (N, C, L)
        t = t.unsqueeze(2)
    p = t.permute(0, 2, 3, 1)
    return p if p.is_contiguous() else p.contiguous()


class _CEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target):
        if not logits.is_cuda:
            raise RuntimeError("atomai_b200 losses run on CUDA (sm_90a) only")
        l = _nhwc_view(logits.detach().float())
        tgt = target.detach()
        if tgt.dtype != torch.int64:
            tgt = tgt.long()
        tgt = tgt.contiguous()
        npix = l.shape[0] * l.shape[1] * l.shape[2]
        assert tgt.numel() == npix, "target shape does not match logits"
        acc = torch.zeros(1, device=l.device, dtype=torch.float64)
        ops.ce_fwd_bwd(l, tgt, acc)
        ctx.save_for_backward(l, tgt)
        ctx.shape, ctx.npix = logits.shape, npix
        return (acc / npix).float().reshape(())

    @staticmethod
    def backward(ctx, g):
        l, tgt = ctx.saved_tensors
        d = torch.empty_like(l)
        ops.ce_fwd_bwd(l, tgt, None, d, 1.0 / ctx.npix, g.detach().float().reshape(1).contiguous())
        gl = d.permute(0, 3, 1, 2)
        if len(ctx.shape) == 3:
            gl = gl.squeeze(2)
        elif len(ctx.shape) == 2:
            gl = gl.reshape(ctx.shape)
        return gl, None


class _PointwiseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, kind):
        if not pred.is_cuda:
            raise RuntimeError("atomai_b200 losses run on CUDA (sm_90a) only")
        # elementwise: memory order is irrelevant as long as both operands share it
        if pred.stride() == target.stride() and pred.is_non_overlapping_and_dense() \
                and target.is_non_overlapping_and_dense():
            p, t = pred.detach(), target.detach()
        else:
            p, t = pred.detach().contiguous(), target.detach().contiguous()
        t = t.float() if t.dtype != torch.float32 else t
        acc = torch.zeros(1, device=p.device, dtype=torch.float64)
        ops.pointwise_loss(p, t, kind, acc)
        ctx.save_for_backward(p, t)
        ctx.kind, ctx.shape, ctx.same = kind, pred.shape, p.stride() == pred.stride()
        return (acc / p.numel()).float().reshape(())

    @staticmethod
    def backward(ctx, g):
        p, t = ctx.saved_tensors
        d = torch.empty_like(p)
        ops.pointwise_loss(p, t, ctx.kind, None, d, 1.0 / p.numel(),
                           g.detach().float().reshape(1).contiguous())
        return d, None, None


class CrossEntropyLoss(torch.nn.CrossEntropyLoss):
    """Mean cross-entropy over (N,C,H,W) logits and (N,H,W) int64 labels, fused fwd/bwd kernel."""
    def forward(self, input, target):
        if self.weight is not None or self.ignore_index != -100 or self.reduction != "mean" \
                or self.label_smoothing != 0.0:
            raise NotImplementedError("native CrossEntropyLoss supports the default options only")
        return _CEFn.apply(input, target)


class BCEWithLogitsLoss(torch.nn.BCEWithLogitsLoss):
    def forward(self, input, target):
        if self.weight is not None or self.pos_weight is not None or self.reduction != "mean":
            raise NotImplementedError("native BCEWithLogitsLoss supports the default options only")
        return _PointwiseFn.apply(input, target, 1)


class MSELoss(torch.nn.MSELoss):
    def forward(self, input, target):
        if self.reduction != "mean":
            raise NotImplementedError("native MSELoss supports reduction='mean' only")
        return _PointwiseFn.apply(input, target, 0)


def select_loss(loss: str, nb_classes: int = None, **kwargs):
    """
    Selects loss for DCNN model training (contract of atomai/losses_metrics/losses.py:139-174).
    'ce' -> CrossEntropyLoss (nb_classes > 2) / BCEWithLogitsLoss (nb_classes == 1), 'mse'.
    'dice' / 'focal' / multitask losses are outside the accelerated hot path (SURVEY.md §2.1).
    """
    if loss in ['ce', 'multitask'] and nb_classes is None:
        raise ValueError("For cross-entropy loss function, you must" +
                         " specify the number of classes")
    if loss == 'ce' and nb_classes == 1:
        criterion = BCEWithLogitsLoss()
    elif loss == 'ce' and nb_classes > 2:
        criterion = CrossEntropyLoss()
    elif loss == 'mse':
        criterion = MSELoss()
    elif hasattr(loss, "__call__"):
        criterion = loss
    else:
        raise NotImplementedError(
            "Select cross-entropy loss ('ce'), means-squared error ('mse')"
            " or pass your custom loss function ('dice', 'focal' and multitask losses are"
            " not part of the atomai_b200 hot path)"
        )
    return criterion
