"""
Segmentation accuracy for the native path: the reference's mean Intersection over Union
(atomai/losses_metrics/metrics.py:16-95) counted on the GPU.  The reference copies the logits to
the host and thresholds them image by image with cv2; here one kernel thresholds every pixel and
builds the confusion histogram (exact int64 counts) and a one-thread kernel applies the
reference's float32 formula, so the metric never leaves the device until it is read.
"""
import torch

from .. import ops


class IoU:
    """
    Mean IoU of a batch (API of atomai/losses_metrics/metrics.py:16-95).

    Args:
        true: labels, (N, H, W) class indices (C > 1) or (N, 1, H, W) binary masks (C == 1)
        pred: model outputs (N, C, H, W) on the GPU
        activation: apply softmax (C > 1) / sigmoid (C == 1) before thresholding
        thresh: binary threshold of the class probabilities (strict: p > thresh)
        comm: data-parallel Comm; the confusion counts are added over the ranks, so the value is
            that of the global batch
    """
    def __init__(self, true: torch.Tensor, pred: torch.Tensor, activation: bool = True,
                 thresh: float = 0.5, comm=None):
        if not pred.is_cuda:
            raise RuntimeError("atomai_b200 metrics run on CUDA (sm_90a) only")
        if pred.dim() != 4:
            raise NotImplementedError("native IoU takes (N, C, H, W) predictions")
        N, C, H, W = pred.shape
        self.thresh = thresh
        self.nb_classes = 2 if C == 1 else C
        t = true.detach().to(pred.device)
        if t.numel() != N * H * W:
            raise ValueError(f"IoU: labels of shape {tuple(true.shape)} do not match predictions "
                             f"of shape {tuple(pred.shape)}")
        if t.dtype not in (torch.int64, torch.float32):
            t = t.float() if t.is_floating_point() else t.long()
        t = t.contiguous()
        p = pred.detach().float().permute(0, 2, 3, 1)
        p = p if p.is_contiguous() else p.contiguous()
        self.counts = torch.zeros(self.nb_classes ** 2, device=pred.device, dtype=torch.int64)
        ops.iou_hist(p, t, thresh, self.counts, activation=bool(activation))
        if comm is not None and comm.world > 1:
            comm.allreduce_any_(self.counts)

    def confusion(self) -> torch.Tensor:
        """(nc, nc) int64 histogram, rows = true class, columns = predicted class."""
        return self.counts.reshape(self.nb_classes, self.nb_classes)

    def evaluate_device(self) -> torch.Tensor:
        """Mean IoU as a 0-d float32 device tensor (no host synchronisation)."""
        out = torch.empty(1, device=self.counts.device, dtype=torch.float32)
        ops.iou_finalize(self.counts, self.nb_classes, out)
        return out.reshape(())

    def evaluate(self) -> float:
        """Computes mean IoU score for a batch (a Python float, as the reference returns)."""
        return self.evaluate_device().item()
