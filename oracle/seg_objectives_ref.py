"""
Torch restatement of the reference's segmentation objectives (CPU or GPU, any float dtype):
dice_loss and focal_loss (atomai/losses_metrics/losses.py:13-89) and the IoU metric
(atomai/losses_metrics/metrics.py:16-95).  Pinned against the reference's own outputs by
tests/test_seg_objectives.py; the GPU tests compare the native kernels with it.
"""
import torch


def dice_cells(logits: torch.Tensor, labels: torch.Tensor):
    """(I, S) per cell, flattened in the reference's order.  Multi-class: softmax over C and
    one-hot (N, H, W) labels, summed over dims (0, 2) -> (C, W) cells (the reference's
    `dims = (0,) + range(2, labels.ndim)` with rank-3 labels: the image rows and the batch, not
    the columns).  C == 1: [sigmoid, 1 - sigmoid] against [y == 1, y == 0], dims (0, 2, 3)."""
    C = logits.shape[1]
    if C == 1:
        y = labels.squeeze(1).long()
        s = torch.sigmoid(logits[:, 0])
        p = torch.stack([s, 1 - s], 1)
        t = torch.stack([(y == 1), (y == 0)], 1).to(logits.dtype)
        dims = (0, 2, 3)
    else:
        p = torch.softmax(logits, 1)
        t = torch.nn.functional.one_hot(labels.long(), C).permute(0, 3, 1, 2).to(logits.dtype)
        dims = (0,) + tuple(range(2, labels.dim()))
    return (p * t).sum(dims).reshape(-1), (p + t).sum(dims).reshape(-1)


def dice_loss(logits: torch.Tensor, labels: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    inter, card = dice_cells(logits, labels)
    return 1 - (2.0 * inter / (card + eps)).mean()


def dice_coefficients(inter: torch.Tensor, card: torch.Tensor, eps: float = 1e-7):
    """(A, B) with dL/dp = t A + B of the dice loss for each cell's probability p and target t:
    A = dL/dI = -(2/K) / (S + eps), B = dL/dS = (2/K) I / (S + eps)^2, K cells."""
    K = inter.numel()
    d = card + eps
    return -(2.0 / K) / d, (2.0 / K) * inter / (d * d)


def focal_loss(logits: torch.Tensor, target: torch.Tensor, alpha: float = 0.5,
               gamma: float = 2.0) -> torch.Tensor:
    """alpha (1 - pt)^gamma CE, CE = mean BCE-with-logits, pt = exp(-CE)."""
    ce = torch.nn.functional.binary_cross_entropy_with_logits(logits, target)
    pt = torch.exp(-ce)
    return alpha * (1 - pt) ** gamma * ce


def focal_factor(ce: torch.Tensor, alpha: float = 0.5, gamma: float = 2.0) -> torch.Tensor:
    """dfocal/dCE = alpha [(1 - pt)^gamma + gamma pt (1 - pt)^(gamma - 1) CE]; the second term is
    dropped for gamma == 0, as autograd does (it is NaN at CE = 0 for 0 < gamma < 1, as there)."""
    pt = torch.exp(-ce)
    q = 1 - pt
    tail = gamma * pt * q ** (gamma - 1) * ce if gamma != 0 else torch.zeros_like(ce)
    return alpha * (q ** gamma + tail)


def iou_counts(true: torch.Tensor, logits: torch.Tensor, thresh: float = 0.5,
               activation: bool = True) -> torch.Tensor:
    """(nc, nc) int64 confusion histogram (rows true, columns predicted) of the reference's IoU:
    predicted class = sum_c c [p_c > thresh], 0 above C - 1; C == 1 -> two classes,
    [sigmoid > thresh]; p = softmax / sigmoid, or the raw values without `activation`; labels
    outside [0, nc) skipped."""
    C = logits.shape[1]
    if C == 1:
        nc = 2
        pred = ((torch.sigmoid(logits[:, 0]) if activation else logits[:, 0]) > thresh).long()
    else:
        nc = C
        m = ((torch.softmax(logits, 1) if activation else logits) > thresh).long()
        cls = torch.arange(C, device=logits.device).reshape(1, C, 1, 1)
        pred = (m * cls).sum(1)
        pred[pred > C - 1] = 0
    y = true.reshape(pred.shape).long()
    ok = (y >= 0) & (y < nc)
    h = torch.bincount((nc * y[ok] + pred[ok]).reshape(-1), minlength=nc * nc)
    return h.reshape(nc, nc)


def iou_from_counts(counts: torch.Tensor) -> float:
    """The reference's float32 finalise: mean of diag / (rowsum + colsum - diag + 1e-10)."""
    hist = counts.float()
    d = torch.diag(hist)
    jcd = d / (hist.sum(1) + hist.sum(0) - d + 1e-10)
    return torch.mean(jcd[jcd == jcd]).item()
