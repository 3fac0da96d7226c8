"""Generate tests/golden/unet_resnet.npz by running the UNMODIFIED reference models/unet.py on oracle-made weights and
synthetic inputs (build container only, like oracle/make_golden.py):

    python -m oracle.make_golden_unet_resnet

Shim (non-invasive): pretrained=False.  UNetResnet has no dropout.
Cases (resnet50, 19 classes, CrossEntropyLoss2d(ignore_index=255)), each a train step (loss, sampled logits, argmax,
gradient norms, selected gradients, BN running statistics) followed by an eval forward with the updated statistics:
  s64/  2x3x64x64: upconv1 / upconv2 are resampled x1/2 to the 8x8 skips, upconv3 already has x1's 16x16 size, upconv5's
        output is 64x64
  s65/  2x3x65x65: every resample runs (18 -> 9, 18 -> 9, 18 -> 17 and the final 68 -> 65)
"""
import os

import numpy as np
import torch

from .make_golden import OUT, import_reference

SMALL_GRADS = ["upconv5.weight", "conv3.bias", "conv7.weight", "initial.0.0.weight"]
BN_TRACK = ["initial.0.1", "initial.1", "layer4.2.bn3"]


def train_step(ref, sd, x, y, crit, prefix, rec):
    ref.load_state_dict(sd, strict=True)  # proves the oracle's key names and shapes are the reference's
    ref.train()
    out = ref(x)
    loss = crit(out, y)
    loss.backward()
    params = dict(ref.named_parameters())
    rec[prefix + "param_names"] = np.array(list(params))
    rec[prefix + "grad_norms"] = np.array([p.grad.double().norm().item() for p in params.values()])
    rec[prefix + "loss"] = np.float64(loss.item())
    rec[prefix + "out_shape"] = np.array(out.shape)
    rec[prefix + "logits_sub"] = out.detach()[:, :, ::4, ::4].numpy()
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
    import models.unet as U
    from oracle import synth, unet_resnet

    rec = {}
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    for prefix, size, seed, xseed in (("s64/", 64, 11, 9011), ("s65/", 65, 12, 9012)):
        sd = unet_resnet.unet_resnet_state_dict(19, seed=seed, randomize_bn=True)
        x, y = synth.make_batch(2, size, size, 19, 255, seed=xseed)
        train_step(U.UNetResnet(19, backbone="resnet50", pretrained=False), sd, x, y, crit, prefix, rec)
    np.savez_compressed(os.path.join(OUT, "unet_resnet.npz"), **rec)
    print("unet_resnet.npz written")


if __name__ == "__main__":
    main()
