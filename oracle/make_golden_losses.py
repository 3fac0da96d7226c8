"""Generate tests/golden/losses_focal_weighted.npz by running the UNMODIFIED reference loss classes (utils/losses.py:24-31
CrossEntropyLoss2d, :52-65 FocalLoss, :67-77 CE_DiceLoss) on synthetic logits, with the import shims of make_golden.py.
Run where a reference checkout exists:

    python -m oracle.make_golden_losses

Records, per case, the reference's loss and its autograd gradient of the logits (NaN where the reference gives NaN: a
mean over nothing valid, and FocalLoss with 0 < gamma < 1 where pt rounds to 1).  Layout: `cases` is a JSON list of
{id, input, kind ('ce' | 'focal' | 'ce_dice'), weight (bool), gamma, reduction}; the inputs are `in/<input>/logits`,
`in/<input>/target`, `in/<input>/ignore` and `in/<input>/weight`; the results are `<id>/loss` and `<id>/grad`
(and `<id>/target_after` for CE_DiceLoss, whose Dice term rewrites the caller's target in place).  With ignored pixels
present that rewrite also hits the target CE saved for its backward, so the reference cannot back-propagate CE_DiceLoss
there: such a case records the loss, NaN gradients and `<id>/backward_error`.
"""
import json
import os
import sys

import numpy as np
import torch

from oracle.make_golden import OUT, ROOT, import_reference

GAMMAS = (0.0, 0.5, 1.0, 2.0, 2.5)


def make_inputs():
    g = torch.Generator().manual_seed(2024)
    ins = {}
    N, H, W = 2, 5, 6
    for C, ign in ((19, 255), (21, 255), (150, -1)):
        logits = torch.randn(N, C, H, W, generator=g) * 3
        target = torch.randint(0, C, (N, H, W), generator=g)
        target[:, 0, :3] = ign
        target[1, 4, :] = ign
        w = torch.rand(C, generator=g) * 2 + 0.1
        w[torch.randperm(C, generator=g)[: max(2, C // 6)]] = 0.0  # some classes weigh nothing
        ins[f"c{C}"] = (logits, target, ign, w)
    logits, target, ign, w = ins["c19"]
    t = target.clone()
    t[1] = ign  # one fully ignored image
    ins["c19_img_ignored"] = (logits, t, ign, w)
    ins["c19_all_ignored"] = (logits, torch.full_like(target, ign), ign, w)  # ATen's mean over nothing: NaN
    t = target.clone()
    t[(t != ign)] = int(torch.nonzero(w == 0)[0])  # every labelled pixel is a zero-weight class: weighted D = 0
    ins["c19_zero_weight"] = (logits, t, ign, w)
    sat = logits.clone()
    sat[:, :, 1:3, :] = 0.0
    sat[:, 0, 1:3, :] = 100.0  # saturated: pt rounds to 1 in fp32 at label 0
    t = target.clone()
    t[:, 1:3, :] = 0
    ins["c19_saturated"] = (sat, t, ign, w)
    t = target.clone()
    t[t == ign] = 3
    ins["c19_no_ignore"] = (logits, t, ign, w)
    return ins


def run(crit, logits, target):
    x = logits.clone().requires_grad_(True)
    t = target.clone()
    loss = crit(x, t)
    try:
        loss.backward()
        return loss.detach(), x.grad.detach(), t, ""
    except RuntimeError as e:
        return loss.detach(), torch.full_like(logits, float("nan")), t, str(e).splitlines()[0][:200]


def main():
    torch.set_num_threads(8)
    _, losses = import_reference()
    sys.path.insert(0, ROOT)
    ins = make_inputs()
    rec, cases = {}, []
    for name, (logits, target, ign, w) in ins.items():
        rec[f"in/{name}/logits"] = logits.numpy()
        rec[f"in/{name}/target"] = target.numpy()
        rec[f"in/{name}/ignore"] = np.int64(ign)
        rec[f"in/{name}/weight"] = w.numpy()
        full = name in ("c19", "c19_saturated")
        gammas = GAMMAS if full else (0.0, 2.0)
        for use_w in (False, True):
            alpha = w if use_w else None
            for red in ("mean", "sum"):
                todo = [("ce", None, losses.CrossEntropyLoss2d(weight=alpha, ignore_index=ign, reduction=red))]
                todo += [("focal", gm, losses.FocalLoss(gamma=gm, alpha=alpha, ignore_index=ign, size_average=red == "mean"))
                         for gm in gammas]
                if name in ("c19", "c19_no_ignore"):
                    todo.append(("ce_dice", None, losses.CE_DiceLoss(weight=alpha, ignore_index=ign, reduction=red)))
                for kind, gm, crit in todo:
                    cid = f"{name}/{kind}/{'w' if use_w else 'now'}/{red}" + ("" if gm is None else f"/g{gm}")
                    loss, grad, t_after, err = run(crit, logits, target)
                    rec[f"{cid}/loss"] = np.float64(loss.item())
                    rec[f"{cid}/grad"] = grad.numpy()
                    if kind == "ce_dice":
                        rec[f"{cid}/target_after"] = t_after.numpy()
                    if err:
                        rec[f"{cid}/backward_error"] = np.array(err)
                    cases.append({"id": cid, "input": name, "kind": kind, "weight": use_w, "gamma": gm, "reduction": red})
    rec["cases"] = np.array(json.dumps(cases))
    path = os.path.join(OUT, "losses_focal_weighted.npz")
    np.savez_compressed(path, **rec)
    nan_g = sum(1 for c in cases if not np.isfinite(rec[c["id"] + "/grad"]).all())
    nan_l = sum(1 for c in cases if not np.isfinite(rec[c["id"] + "/loss"]))
    print(f"{path}: {len(cases)} cases ({nan_l} NaN losses, {nan_g} with NaN gradients), {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
