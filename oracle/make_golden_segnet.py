"""Generate tests/golden/segnet.npz by running the UNMODIFIED reference models/segnet.py on oracle-made weights and
synthetic inputs (build container only, like oracle/make_golden.py):

    python -m oracle.make_golden_segnet

Shim (non-invasive, mandatory): the reference constructor always asks torchvision for ImageNet weights
(segnet.py:16, whatever `pretrained` says); `torchvision.models.vgg16_bn` is replaced by a weights=None build BEFORE the
constructor runs, so nothing is downloaded.  SegNet has no dropout.
Cases (19 classes, CrossEntropyLoss2d(ignore_index=255)), each a train step (loss, sampled logits, argmax, gradient norms,
selected gradients, BN running statistics) followed by an eval forward with the updated statistics:
  s64/     2x3x64x64: every pool input is even
  s50x75/  2x3x50x75: odd rows / columns are dropped by several pools on each axis (heights 50 -> 25 -> 12 -> 6 -> 3 -> 1,
           widths 75 -> 37 -> 18 -> 9 -> 4 -> 2) and the unpools write zeros there
"""
import os

import numpy as np
import torch

from .make_golden import OUT, import_reference

SMALL_GRADS = ["stage5_decoder.6.weight", "stage5_decoder.6.bias", "stage1_encoder.0.weight", "stage3_decoder.7.weight",
               "stage5_encoder.6.bias"]
BN_TRACK = ["stage1_encoder.1", "stage5_encoder.7", "stage2_decoder.7", "stage5_decoder.4"]
CASES = (("s64/", 64, 64, 21, 9021), ("s50x75/", 50, 75, 22, 9022))


def install_vgg_shim():
    """torchvision.models.vgg16_bn -> the same network built with weights=None (segnet.py:16 calls it by attribute)."""
    import torchvision
    orig = torchvision.models.vgg16_bn
    if getattr(orig, "_weights_none_shim", False):
        return

    def vgg16_bn(*args, **kwargs):
        kwargs["weights"] = None
        return orig(*args, **kwargs)

    vgg16_bn._weights_none_shim = True
    torchvision.models.vgg16_bn = vgg16_bn


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
    install_vgg_shim()
    models, losses = import_reference()
    import models.segnet as S
    from oracle import segnet, synth

    rec = {}
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    for prefix, h, w, seed, xseed in CASES:
        sd = segnet.segnet_state_dict(19, seed=seed, randomize_bn=True)
        x, y = synth.make_batch(2, h, w, 19, 255, seed=xseed)
        train_step(S.SegNet(19, pretrained=False), sd, x, y, crit, prefix, rec)
    np.savez_compressed(os.path.join(OUT, "segnet.npz"), **rec)
    print("segnet.npz written")


if __name__ == "__main__":
    main()
