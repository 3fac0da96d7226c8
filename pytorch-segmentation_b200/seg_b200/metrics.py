"""`utils.metrics` of the reference behind one device pass (SURVEY.md §8f rank 1).

`eval_metrics(output, target, num_class)` — utils/metrics.py:59-67 — is called on every training step
(trainer.py:84) and costs the reference an argmax pass, three histc passes and four `.cpu()` syncs over the full-size
logits.  Here: one kernel (argmax + pixel accuracy + per-class intersection / prediction / label histograms, integer
counters) and ONE small device-to-host copy.  Return value and rounding are the reference's.
"""
import numpy as np
import torch

from . import ops


def eval_metrics(output, target, num_class):
    if not output.is_cuda:
        raise RuntimeError("seg_b200.eval_metrics runs on an H100 only; there is no CPU fallback")
    v = ops.eval_metrics_nchw(output.detach().contiguous().float(), target.contiguous(), num_class).cpu().numpy()
    K = num_class
    correct, labeled = v[0], v[1]
    inter = v[2:2 + K].astype(np.float32)
    union = (v[2 + K:2 + 2 * K] + v[2 + 2 * K:2 + 3 * K] - v[2:2 + K]).astype(np.float32)
    assert correct <= labeled, "Correct area should be smaller than Labeled"
    assert (inter <= union).all(), "Intersection area should be smaller than Union area"
    return [np.round(np.asarray(correct), 5), np.round(np.asarray(labeled), 5), np.round(inter, 5), np.round(union, 5)]


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
