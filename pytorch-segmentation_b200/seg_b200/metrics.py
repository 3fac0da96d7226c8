"""`utils.metrics` of the reference behind one device pass (SURVEY.md §8f rank 1).

`eval_metrics(output, target, num_class)` — utils/metrics.py:59-67 — is called on every training step
(trainer.py:84) and costs the reference an argmax pass, three histc passes and four `.cpu()` syncs over the full-size
logits.  Here: one kernel (argmax + pixel accuracy + per-class intersection / prediction / label histograms, integer
counters) and ONE small device-to-host copy.  Return value and rounding are the reference's.
"""
import numpy as np
import torch

from . import ops


def counters_to_values(v, num_class):
    """Counter vector [2 + 3K] (eval_metrics_nchw, FusedTrainStep.seg_counters) -> (correct, labeled, inter[K], union[K]),
    exact int64, with the reference's sanity checks (utils/metrics.py:45,56)."""
    K = num_class
    v = np.asarray(v, dtype=np.int64)
    correct, labeled = v[0], v[1]
    inter = v[2:2 + K]
    union = v[2 + K:2 + 2 * K] + v[2 + 2 * K:2 + 3 * K] - inter
    assert correct <= labeled, "Correct area should be smaller than Labeled"
    assert (inter <= union).all(), "Intersection area should be smaller than Union area"
    return correct, labeled, inter, union


def eval_metrics(output, target, num_class):
    if not output.is_cuda:
        raise RuntimeError("seg_b200.eval_metrics runs on an H100 only; there is no CPU fallback")
    v = ops.eval_metrics_nchw(output.detach().contiguous().float(), target.contiguous(), num_class).cpu().numpy()
    correct, labeled, inter, union = counters_to_values(v, num_class)
    inter, union = inter.astype(np.float32), union.astype(np.float32)  # torch.histc's dtype
    return [np.round(np.asarray(correct), 5), np.round(np.asarray(labeled), 5), np.round(inter, 5), np.round(union, 5)]


def seg_metrics(counters, num_class):
    """Trainer._get_seg_metrics (trainer.py:186-194) on running totals held as a counter vector [2 + 3K]: Pixel_Accuracy,
    Mean_IoU and Class_IoU, with np.spacing(1) and the 3-decimal rounding.

    One deliberate difference: the reference sums each batch's float32 `inter` / `union` into float32 running totals
    (Trainer._update_seg_metrics), which stop being exact once a class passes 2**24 pixels; the totals here are exact
    int64 counts, converted to float64 only for the ratios."""
    correct, labeled, inter, union = counters_to_values(counters, num_class)
    pix_acc = 1.0 * correct / (np.spacing(1) + labeled)
    iou = 1.0 * inter / (np.spacing(1) + union)
    return {"Pixel_Accuracy": np.round(pix_acc, 3), "Mean_IoU": np.round(iou.mean(), 3),
            "Class_IoU": dict(zip(range(num_class), np.round(iou, 3)))}


class AverageMeter(object):
    """Running weighted average (utils/metrics.py:6-39): same attributes and update rule."""

    def __init__(self):
        self.initialized = False
        self.val = self.avg = self.sum = self.count = None

    def update(self, val, weight=1):
        if not self.initialized:
            self.val, self.avg, self.sum, self.count, self.initialized = val, val, np.multiply(val, weight), weight, True
        else:
            self.val = val
            self.sum = np.add(self.sum, np.multiply(val, weight))
            self.count = self.count + weight
            self.avg = self.sum / self.count

    @property
    def value(self):
        return self.val

    @property
    def average(self):
        return np.round(self.avg, 5)
