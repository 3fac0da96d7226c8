"""Drop-in losses for the reference's loss registry (`getattr(losses, config['loss'])(ignore_index=...)`, train.py:30).

    CrossEntropyLoss2d(weight=None, ignore_index=255, reduction='mean')   — utils/losses.py:24-31
    DiceLoss(smooth=1., ignore_index=255)                                 — utils/losses.py:33-50
    CE_DiceLoss(smooth=1, reduction='mean', ignore_index=255, weight=None) — utils/losses.py:67-77
    LovaszSoftmax(classes='present', per_image=False, ignore_index=255)   — utils/losses.py:79-89

forward(output fp32 [B,C,H,W], target int64 [B,H,W]) -> 0-dim tensor with autograd, computed by the sm_90a kernels
(`seg_ce_nchw_fwd/bwd`); `.item()` works as the trainer expects (trainer.py:72,81).  CUDA tensors only.
"""
import torch
import torch.nn as nn

from . import ops


def _dp_world():
    from .comm import dp_world
    return dp_world()


class _CEFn(torch.autograd.Function):
    """mean over the non-ignored pixels (nn.CrossEntropyLoss(reduction='mean', ignore_index), utils/losses.py:24-31).  In the
    reference nn.DataParallel gathers the logits and the loss is the mean over the GLOBAL batch; with one process per GPU
    that is (sum over ranks of the loss sums) / (sum over ranks of the valid-pixel counts): the (sum, count) pair is
    all-reduced — 16 bytes — so every rank reports the global loss and its gradient carries the global normalisation
    (times world: the engine's gradient exchange averages over ranks).  `global_mean=False` keeps per-rank means."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, global_mean=True):
        logits = logits.contiguous().float()
        target = target.contiguous()
        world = _dp_world() if global_mean else 1
        reduce_fn = None
        if world > 1:
            def reduce_fn(accum):
                torch.distributed.all_reduce(accum)
        loss, accum = ops.ce_nchw_fwd(logits, target, ignore_index, reduce_fn=reduce_fn)
        ctx.save_for_backward(logits, target, accum)
        ctx.ignore_index, ctx.world = ignore_index, world
        return loss

    @staticmethod
    def backward(ctx, gout):
        logits, target, accum = ctx.saved_tensors
        g = gout.detach().reshape(1).float().contiguous()
        if ctx.world > 1:
            g = g * float(ctx.world)
        return (ops.ce_nchw_bwd(logits, target, ctx.ignore_index, accum, gscale=g),) + (None,) * (len(ctx.needs_input_grad) - 1)


class CrossEntropyLoss2d(nn.Module):
    def __init__(self, weight=None, ignore_index=255, reduction="mean"):
        super().__init__()
        if weight is not None or reduction != "mean":
            raise NotImplementedError("seg_b200.CrossEntropyLoss2d: only weight=None, reduction='mean' (the configs' setting)")
        self.ignore_index = ignore_index

    def forward(self, output, target):
        if not output.is_cuda:
            raise RuntimeError("seg_b200 losses run on an H100 only; there is no CPU fallback")
        return _CEFn.apply(output, target, self.ignore_index)


class _DiceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, smooth):
        logits = logits.contiguous().float()
        loss, accum = ops.dice_nchw_fwd(logits, target, smooth)
        ctx.save_for_backward(logits, target, accum)
        ctx.smooth = smooth
        return loss

    @staticmethod
    def backward(ctx, gout):
        logits, target, accum = ctx.saved_tensors
        g = gout.detach().reshape(1).float().contiguous()
        return ops.dice_nchw_bwd(logits, target, accum, ctx.smooth, gscale=g), None, None


def _dice_fix_target_(target, ignore_index):
    """The reference's label fix-up, reproduced including its in-place mutation of the caller's tensor and its
    `range(min, max)` test (utils/losses.py:40-42): ignored pixels become target.min()."""
    tmin, tmax = int(target.min()), int(target.max())
    if ignore_index not in range(tmin, tmax):
        if (target == ignore_index).sum() > 0:
            target[target == ignore_index] = tmin
    return target


class DiceLoss(nn.Module):
    def __init__(self, smooth=1.0, ignore_index=255):
        super().__init__()
        self.ignore_index = ignore_index
        self.smooth = smooth

    def forward(self, output, target):
        if not output.is_cuda:
            raise RuntimeError("seg_b200 losses run on an H100 only; there is no CPU fallback")
        target = _dice_fix_target_(target, self.ignore_index)
        return _DiceFn.apply(output, target.contiguous(), float(self.smooth))


class CE_DiceLoss(nn.Module):
    def __init__(self, smooth=1, reduction="mean", ignore_index=255, weight=None):
        super().__init__()
        if weight is not None or reduction != "mean":
            raise NotImplementedError("seg_b200.CE_DiceLoss: only weight=None, reduction='mean'")
        self.smooth = smooth
        self.dice = DiceLoss()  # the reference builds it with the DEFAULT ignore_index (utils/losses.py:71)
        self.ignore_index = ignore_index

    def forward(self, output, target):
        ce = _CEFn.apply(output, target, self.ignore_index)  # CE first: it sees the target before Dice mutates it
        return ce + self.dice(output, target)


class _LovaszFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index):
        loss, dl = ops.lovasz_softmax_nchw(logits.contiguous().float(), target.contiguous(), ignore_index)
        ctx.save_for_backward(dl)
        return loss

    @staticmethod
    def backward(ctx, gout):
        (dl,) = ctx.saved_tensors
        return dl * gout, None, None


class LovaszSoftmax(nn.Module):
    def __init__(self, classes="present", per_image=False, ignore_index=255):
        super().__init__()
        if classes != "present" or per_image:
            raise NotImplementedError("seg_b200.LovaszSoftmax: classes='present', per_image=False (the configs' setting)")
        self.smooth = classes  # the reference stores `classes` under this (unused) name, utils/losses.py:82
        self.per_image = per_image
        self.ignore_index = ignore_index

    def forward(self, output, target):
        if not output.is_cuda:
            raise RuntimeError("seg_b200 losses run on an H100 only; there is no CPU fallback")
        return _LovaszFn.apply(output, target, self.ignore_index)
