"""
Loss functions for the native path.  `select_loss` has the reference's contract
(atomai/losses_metrics/losses.py:139-174): the returned criteria are nn.Modules whose names and
reprs match the reference's (`str(criterion) == "CrossEntropyLoss()"` / `"dice_loss()"`,
test/trainers/test_trainer.py:59-74) but whose forward/backward run as fused sm_90a kernels: one
pass computes the summed loss, the backward pass recomputes the softmax and writes d(logits)
scaled by the upstream gradient read from device memory (no host synchronisation).
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


def _world(comm) -> int:
    return comm.world if comm is not None else 1


class _DiceFn(torch.autograd.Function):
    """Dice loss of (N, C, H, W) logits: per-cell (I, S) sums, device finalise, elementwise
    backward.  Under data parallelism (`comm`) the cell sums are added over the ranks before the
    finalise, so loss and gradients are those of the global batch; the gradient is scaled by the
    world size because the trainer averages the summed parameter gradients over the ranks."""
    @staticmethod
    def forward(ctx, logits, target, eps, comm):
        if not logits.is_cuda:
            raise RuntimeError("atomai_b200 losses run on CUDA (sm_90a) only")
        if logits.dim() != 4:
            raise NotImplementedError("native dice_loss takes (N, C, H, W) logits")
        N, C, H, W = logits.shape
        tgt = target.detach()
        if C > 1:
            if tgt.shape != (N, H, W):
                raise NotImplementedError("native dice_loss takes (N, H, W) labels for C > 1")
            tgt = tgt.long()
        else:
            if tgt.shape != (N, 1, H, W):
                raise NotImplementedError("native dice_loss takes (N, 1, H, W) labels for C == 1")
            if tgt.dtype not in (torch.float32, torch.int64):
                tgt = tgt.float() if tgt.is_floating_point() else tgt.long()
        tgt = tgt.contiguous()
        l = _nhwc_view(logits.detach().float())
        K = 2 if C == 1 else C * W
        cells = torch.empty(2 * K, device=l.device, dtype=torch.float64)
        ops.dice_sums(l, tgt, cells)
        if _world(comm) > 1:
            comm.allreduce_any_(cells)
        loss = torch.empty(1, device=l.device, dtype=torch.float32)
        coef = torch.empty(2 * K, device=l.device, dtype=torch.float32)
        ops.dice_finalize(cells, eps, loss, coef)
        ctx.save_for_backward(l, tgt, coef)
        ctx.world = _world(comm)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        l, tgt, coef = ctx.saved_tensors
        d = torch.empty_like(l)
        ops.dice_bwd(l, tgt, coef, d, float(ctx.world), g.detach().float().reshape(1).contiguous())
        return d.permute(0, 3, 1, 2), None, None, None


class _FocalFn(torch.autograd.Function):
    """Focal loss of logits: the BCE-with-logits sum (pointwise_loss kind 1), then the scalar
    transform and its derivative factor on the device; backward is the BCE gradient scaled by
    factor / count.  Data parallel: the BCE sum and the count are global (see _DiceFn)."""
    @staticmethod
    def forward(ctx, pred, target, alpha, gamma, comm):
        if not pred.is_cuda:
            raise RuntimeError("atomai_b200 losses run on CUDA (sm_90a) only")
        if pred.shape != target.shape:
            raise ValueError(f"focal_loss: target shape {tuple(target.shape)} != input shape "
                             f"{tuple(pred.shape)}")
        p, t = pred.detach().float().contiguous(), target.detach().float().contiguous()
        acc = torch.zeros(1, device=p.device, dtype=torch.float64)
        ops.pointwise_loss(p, t, 1, acc)
        world = _world(comm)
        if world > 1:
            comm.allreduce_any_(acc)
        count = p.numel() * world
        loss = torch.empty(1, device=p.device, dtype=torch.float32)
        factor = torch.empty(1, device=p.device, dtype=torch.float32)
        ops.focal_finalize(acc, count, alpha, gamma, loss, factor)
        ctx.save_for_backward(p, t, factor)
        ctx.gscale = world / count
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        p, t, factor = ctx.saved_tensors
        d = torch.empty_like(p)
        ops.pointwise_loss(p, t, 1, None, d, ctx.gscale,
                           (g.detach().float().reshape(1) * factor).contiguous())
        return d, None, None, None, None


class dice_loss(torch.nn.Module):
    """Sørensen–Dice loss of the reference (atomai/losses_metrics/losses.py:53-89), including its
    reduction: for (N, H, W) labels the sums run over dims (0, 2), one cell per (class, image
    column), and the loss is 1 - the mean of 2 I / (S + eps) over those cells."""
    def __init__(self, eps: float = 1e-7):
        super(dice_loss, self).__init__()
        self.eps = eps
        self.comm = None       # data-parallel Comm, set by the trainer

    def forward(self, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        return _DiceFn.apply(logits, labels, self.eps, self.comm)


class focal_loss(torch.nn.Module):
    """Focal loss of the reference (losses.py:13-50): alpha (1 - pt)^gamma CE with CE the mean
    BCE-with-logits and pt = exp(-CE).  Logits only."""
    def __init__(self, alpha: float = 0.5, gamma: float = 2, with_logits: bool = True) -> None:
        super(focal_loss, self).__init__()
        if not with_logits:
            raise NotImplementedError("native focal_loss takes logits (with_logits=True) only")
        self.alpha = alpha
        self.gamma = gamma
        self.logits = with_logits
        self.comm = None       # data-parallel Comm, set by the trainer

    def forward(self, prediction: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        return _FocalFn.apply(prediction, labels, float(self.alpha), float(self.gamma), self.comm)


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
    'dice' -> dice_loss, 'focal' -> focal_loss, 'ce' -> CrossEntropyLoss (nb_classes > 2) /
    BCEWithLogitsLoss (nb_classes == 1), 'mse'.  Multitask losses are outside the accelerated hot
    path (SURVEY.md §2.1).
    """
    if loss in ['ce', 'multitask'] and nb_classes is None:
        raise ValueError("For cross-entropy loss function, you must" +
                         " specify the number of classes")
    if loss == 'dice':
        criterion = dice_loss()
    elif loss == 'focal':
        criterion = focal_loss()
    elif loss == 'ce' and nb_classes == 1:
        criterion = BCEWithLogitsLoss()
    elif loss == 'ce' and nb_classes > 2:
        criterion = CrossEntropyLoss()
    elif loss == 'mse':
        criterion = MSELoss()
    elif hasattr(loss, "__call__"):
        criterion = loss
    else:
        raise NotImplementedError(
            "Select Dice loss ('dice'), focal loss ('focal'), cross-entropy loss ('ce'),"
            " means-squared error ('mse') or pass your custom loss function (multitask losses"
            " are not part of the atomai_b200 hot path)"
        )
    return criterion
