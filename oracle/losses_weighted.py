"""CPU restatement of the reference's class-weighted and focal losses (TEST INFRASTRUCTURE).

  cross_entropy2d -> utils/losses.py:24-31 (nn.CrossEntropyLoss(weight, ignore_index, reduction))
  focal_loss      -> utils/losses.py:52-65 (as written: autograd through it has the reference's NaN where pt rounds to 1)
  focal_grad_factor, weighted_loss_and_grad -> float64 loss and logits gradient of the class-weighted CE / focal loss as
                     the engine defines them (finite limit where pt rounds to 1, 0 for a mean over a zero denominator)

CE_DiceLoss(weight, reduction) (utils/losses.py:67-77) is weighted_loss_and_grad's CE plus oracle.losses.dice_loss.
"""
import torch
import torch.nn.functional as F


def cross_entropy2d(output, target, ignore_index=255, weight=None, reduction="mean"):
    return F.cross_entropy(output, target, weight=weight, ignore_index=ignore_index, reduction=reduction)


def focal_loss(output, target, gamma=2, alpha=None, ignore_index=255, size_average=True):
    logpt = F.cross_entropy(output, target, weight=alpha, ignore_index=ignore_index, reduction="none")
    pt = torch.exp(-logpt)
    loss = ((1 - pt) ** gamma) * logpt
    return loss.mean() if size_average else loss.sum()


def focal_grad_factor(L, gamma):
    """dF/dL of F(L) = (1 - exp(-L))^gamma * L, as u^gamma * (1 + gamma * r) with u = -expm1(-L) and r = L / expm1(L)
    (r = 1 at L = 0): u and r lie in [0, 1], so 0 <= F' <= 1 + gamma, and no 0 * inf is formed at L = 0."""
    u = -torch.expm1(-L)
    r = torch.where(L > 0, L / torch.expm1(L), torch.ones_like(L))
    return u ** gamma * (1 + gamma * r)


def weighted_loss_and_grad(output, target, ignore_index=255, weight=None, gamma=None, mean=True):
    """float64 (loss, d loss / d output) for CrossEntropyLoss2d(weight, reduction) (gamma None) or FocalLoss(gamma,
    alpha=weight, size_average=mean).  Denominator of a mean: the sum of the valid pixels' class weights (CE) or every
    pixel (focal); a mean over a zero denominator is 0 with gradient 0 (ATen gives NaN)."""
    z = output.detach().double()
    C = z.shape[1]
    valid = target != ignore_index
    t = torch.where(valid, target, torch.zeros_like(target))
    nll = torch.logsumexp(z, 1) - z.gather(1, t.unsqueeze(1)).squeeze(1)
    dev = z.device
    w = torch.ones(C, dtype=torch.float64, device=dev) if weight is None else torch.as_tensor(weight, dtype=torch.float64).to(dev)
    wt = w[t] * valid
    L = wt * nll
    if gamma is None:
        per, fac, D = L, wt, wt.sum()
    else:
        per, fac, D = (-torch.expm1(-L)) ** gamma * L, wt * focal_grad_factor(L, gamma), torch.tensor(float(target.numel()), dtype=torch.float64, device=dev)
    if mean:
        g = 1.0 / D if D > 0 else torch.zeros((), dtype=torch.float64, device=dev)
    else:
        g = torch.ones((), dtype=torch.float64, device=dev)
    loss = per.sum() * g
    onehot = F.one_hot(t, C).permute(0, 3, 1, 2).double()
    grad = g * (fac * valid).unsqueeze(1) * (F.softmax(z, 1) - onehot)
    return loss, grad
