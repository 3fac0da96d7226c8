"""Drop-in losses for the reference's loss registry (`getattr(losses, config['loss'])(ignore_index=...)`, train.py:30).

    CrossEntropyLoss2d(weight=None, ignore_index=255, reduction='mean')   — utils/losses.py:24-31
    DiceLoss(smooth=1., ignore_index=255)                                 — utils/losses.py:33-50
    FocalLoss(gamma=2, alpha=None, ignore_index=255, size_average=True)   — utils/losses.py:52-65
    CE_DiceLoss(smooth=1, reduction='mean', ignore_index=255, weight=None) — utils/losses.py:67-77
    LovaszSoftmax(classes='present', per_image=False, ignore_index=255)   — utils/losses.py:79-89

forward(output fp32 [B,C,H,W], target int64 [B,H,W]) -> 0-dim tensor with autograd, computed by the sm_90a kernels
(`seg_loss_nchw_fwd/bwd` for cross-entropy, class-weighted CE and focal, `seg_dice_nchw_*`, `seg_lovasz_*`); `.item()` works
as the trainer expects (trainer.py:72,81).  CUDA tensors only.
"""
import torch
import torch.nn as nn

from . import ops


def _dp_world():
    from .comm import dp_world
    return dp_world()


class LossSpec:
    """A cross-entropy (gamma None) or focal loss (gamma >= 0): the class weights (float64 CPU tensor or None = all ones),
    gamma, and whether the loss is a mean (else a sum); ops._loss_kind picks the kernels.  Shared by the plugin path and
    FusedTrainStep."""

    def __init__(self, weight, gamma, mean):
        self.weight, self.gamma, self.mean = weight, gamma, mean
        self._dev = {}

    def weight_on(self, device, C):
        """fp32 [C] copy of the weights on `device` (kept: graph captures bake in its address), or None."""
        if self.weight is None:
            return None
        if self.weight.numel() != C:
            raise ValueError(f"class weight has {self.weight.numel()} entries but the logits have {C} classes")
        key = str(device)
        if key not in self._dev:
            self._dev[key] = self.weight.to(device=device, dtype=torch.float32)
        return self._dev[key]


def _class_weight(weight):
    """`weight` (a sequence or a 1-D tensor) as a float64 CPU tensor; class weights must be finite and >= 0."""
    if weight is None:
        return None
    w = torch.as_tensor(weight).detach().to("cpu", torch.float64).contiguous()
    if w.dim() != 1 or w.numel() == 0:
        raise ValueError(f"class weight must be a non-empty 1-D sequence, got shape {tuple(w.shape)}")
    if not bool(torch.isfinite(w).all()) or bool((w < 0).any()):
        raise ValueError("class weights must be finite and >= 0")
    return w


def _reduction_mean(reduction, name):
    if reduction == "none":
        raise NotImplementedError(f"seg_b200.{name}: reduction='none' is not supported (only 'mean' and 'sum')")
    if reduction not in ("mean", "sum"):
        raise ValueError(f"seg_b200.{name}: reduction must be 'mean' or 'sum', got {reduction!r}")
    return reduction == "mean"


class _CEFn(torch.autograd.Function):
    """mean over the non-ignored pixels (nn.CrossEntropyLoss(reduction='mean', ignore_index), utils/losses.py:24-31).  In the
    reference nn.DataParallel gathers the logits and the loss is the mean over the GLOBAL batch; with one process per GPU
    that is (sum over ranks of the loss sums) / (sum over ranks of the valid-pixel counts): the (sum, count) pair is
    all-reduced — 16 bytes — so every rank reports the global loss and its gradient carries the global normalisation
    (times world: the engine's gradient exchange averages over ranks).  `global_mean=False` keeps per-rank means.
    spec (LossSpec, None = unweighted mean CE): a class-weighted or focal loss instead; its (sum, denominator) pair is
    all-reduced the same way, and a 'sum' is the global sum."""

    @staticmethod
    def forward(ctx, logits, target, ignore_index, global_mean=True, spec=None):
        logits = logits.contiguous().float()
        target = target.contiguous()
        world = _dp_world() if global_mean else 1
        reduce_fn = None
        if world > 1:
            def reduce_fn(accum):
                torch.distributed.all_reduce(accum)
        spec = LossSpec(None, None, True) if spec is None else spec
        loss, accum = ops.loss_nchw_fwd(logits, target, ignore_index, spec.weight_on(logits.device, logits.shape[1]),
                                        spec.gamma, spec.mean, reduce_fn=reduce_fn)
        ctx.save_for_backward(logits, target, accum)
        ctx.ignore_index, ctx.world, ctx.spec = ignore_index, world, spec
        return loss

    @staticmethod
    def backward(ctx, gout):
        logits, target, accum = ctx.saved_tensors
        g = gout.detach().reshape(1).float().contiguous()
        if ctx.world > 1:
            g = g * float(ctx.world)
        spec = ctx.spec
        dl = ops.loss_nchw_bwd(logits, target, ctx.ignore_index, accum, spec.weight_on(logits.device, logits.shape[1]),
                               spec.gamma, spec.mean, gscale=g)
        return (dl,) + (None,) * (len(ctx.needs_input_grad) - 1)


class CrossEntropyLoss2d(nn.Module):
    """weight: per-class weights (sequence or 1-D tensor, finite, >= 0; length checked against C at forward);
    reduction 'mean' (sum of w_t * nll over sum of w_t, 0 when that is 0) or 'sum'."""

    def __init__(self, weight=None, ignore_index=255, reduction="mean"):
        super().__init__()
        mean = _reduction_mean(reduction, "CrossEntropyLoss2d")
        w = _class_weight(weight)
        self.ignore_index = ignore_index
        self.reduction = reduction
        self.spec = LossSpec(w, None, mean)

    def forward(self, output, target):
        if not output.is_cuda:
            raise RuntimeError("seg_b200 losses run on an H100 only; there is no CPU fallback")
        return _CEFn.apply(output, target, self.ignore_index, True, self.spec)


class FocalLoss(nn.Module):
    """utils/losses.py:52-65: (1 - pt)^gamma * L per pixel with L = alpha_t * nll and pt = exp(-L) (not the class
    probability when alpha is set); ignored pixels contribute 0 but size_average=True divides by EVERY pixel, as the
    reference's .mean() of the unreduced loss does.  Where pt rounds to 1 the gradient is its finite limit (0 for
    gamma > 0), not the reference's NaN (DESIGN.md §4)."""

    def __init__(self, gamma=2, alpha=None, ignore_index=255, size_average=True):
        super().__init__()
        gamma = float(gamma)
        if not (gamma >= 0.0 and gamma < float("inf")):
            raise ValueError(f"seg_b200.FocalLoss: gamma must be finite and >= 0, got {gamma}")
        self.gamma = gamma
        self.size_average = size_average
        self.ignore_index = ignore_index
        self.spec = LossSpec(_class_weight(alpha), gamma, bool(size_average))

    def forward(self, output, target):
        if not output.is_cuda:
            raise RuntimeError("seg_b200 losses run on an H100 only; there is no CPU fallback")
        return _CEFn.apply(output, target, self.ignore_index, True, self.spec)


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
        self.cross_entropy = CrossEntropyLoss2d(weight=weight, ignore_index=ignore_index, reduction=reduction)
        self.smooth = smooth
        self.dice = DiceLoss()  # the reference builds it with the DEFAULT ignore_index (utils/losses.py:71)
        self.ignore_index = ignore_index

    def forward(self, output, target):
        ce = self.cross_entropy(output, target)  # CE first: it sees the target before Dice mutates it
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
