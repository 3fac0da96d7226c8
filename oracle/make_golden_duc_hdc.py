"""Generate tests/golden/duc_hdc.npz by running the UNMODIFIED reference models/duc_hdc.py on oracle-made weights and synthetic
inputs (build container only, like oracle/make_golden.py):

    python -m oracle.make_golden_duc_hdc

Shims (non-invasive): the module globals `freeze_backbone` / `set_trainable` that duc_hdc.py:225 reads but never defines
(its constructor raises NameError without them), pretrained=False, dropout p=0 for train parity.
Cases:
  os8/   output_stride=8, 2x3x64x64, 19 classes: train step with CrossEntropyLoss2d (logits, argmax, loss, gradient norms,
         selected gradients, BN running statistics) + an eval forward with the updated statistics
  odd65/ 2x3x65x65, forward only (eval): the output is 68x68 (4 x the 17x17 layer1 size), not cropped to the input
  os4/   output_stride=4, 2x3x32x32: train step (the output is twice the input size)
"""
import os
import sys

import numpy as np
import torch

from .make_golden import OUT, ROOT, import_reference, no_dropout

SMALL_GRADS = ["DUC_out.conv.weight", "DUC_out.bn.weight", "decoder.output.7.bias", "decoder.DUC.bn.weight",
               "ASSP.aspp6.1.weight", "backbone.layer3.22.bn2.bias", "backbone.layer0.0.weight"]
BN_TRACK = ["backbone.layer0.1", "ASSP.avg_pool.2", "decoder.DUC.bn", "DUC_out.bn"]


def train_step(ref, sd, x, y, crit, prefix, rec):
    ref.load_state_dict(sd, strict=True)  # proves the oracle's key names and shapes are the reference's
    no_dropout(ref)
    ref.train()
    out = ref(x)
    loss = crit(out, y)
    loss.backward()
    params = dict(ref.named_parameters())
    rec[prefix + "param_names"] = np.array(list(params))
    rec[prefix + "grad_norms"] = np.array([p.grad.double().norm().item() for p in params.values()])
    rec[prefix + "loss"] = np.float64(loss.item())
    rec[prefix + "out_shape"] = np.array(out.shape)
    rec[prefix + "logits_sub"] = out.detach()[:, :, ::3, ::3].numpy()
    rec[prefix + "logits_sum"] = out.detach().double().sum((2, 3)).numpy()
    rec[prefix + "argmax"] = out.detach().argmax(1).to(torch.uint8).numpy()
    for n in SMALL_GRADS:
        rec[prefix + "grad/" + n] = params[n].grad.numpy()
    rs = ref.state_dict()
    for n in BN_TRACK:
        rec[prefix + "rm/" + n] = rs[n + ".running_mean"].numpy()
        rec[prefix + "rv/" + n] = rs[n + ".running_var"].numpy()
    ref.eval()
    with torch.no_grad():
        rec[prefix + "eval_logits_sum"] = ref(x).double().sum((2, 3)).numpy()
    print(prefix, "loss", loss.item(), "out", tuple(out.shape), "params", len(params))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_num_threads(8)
    models, losses = import_reference()
    import models.duc_hdc as D
    from utils import helpers
    D.freeze_backbone = False
    D.set_trainable = helpers.set_trainable
    sys.path.insert(0, ROOT)
    from oracle import duc_hdc, synth

    rec = {}
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    sd = duc_hdc.duc_hdc_state_dict(19, seed=7, randomize_bn=True)
    x, y = synth.make_batch(2, 64, 64, 19, 255, seed=9005)
    train_step(D.DeepLab_DUC_HDC(19, pretrained=False), sd, x, y, crit, "os8/", rec)

    ref = D.DeepLab_DUC_HDC(19, pretrained=False)
    ref.load_state_dict(sd, strict=True)
    ref.eval()
    x65, _ = synth.make_batch(2, 65, 65, 19, 255, seed=9006)
    with torch.no_grad():
        out = ref(x65)
    rec["odd65/out_shape"] = np.array(out.shape)
    rec["odd65/logits_sum"] = out.double().sum((2, 3)).numpy()
    rec["odd65/logits_sub"] = out[:, :, ::3, ::3].numpy()
    print("odd65/ out", tuple(out.shape))

    sd4 = duc_hdc.duc_hdc_state_dict(19, seed=8, randomize_bn=True)
    x4, y4 = synth.make_batch(2, 32, 32, 19, 255, seed=9007)
    y4 = torch.nn.functional.interpolate(y4[:, None].float(), size=(64, 64), mode="nearest")[:, 0].long()  # output is 2x the input
    train_step(D.DeepLab_DUC_HDC(19, pretrained=False, output_stride=4), sd4, x4, y4, crit, "os4/", rec)
    np.savez_compressed(os.path.join(OUT, "duc_hdc.npz"), **rec)
    print("duc_hdc.npz written")


if __name__ == "__main__":
    main()
