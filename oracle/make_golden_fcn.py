"""Generate tests/golden/fcn.npz by running the UNMODIFIED reference models/fcn.py on oracle-made weights and synthetic
inputs (build container only, like oracle/make_golden.py):

    python -m oracle.make_golden_fcn

Shims (non-invasive, mandatory):
  * the reference constructor asks torchvision for ImageNet weights (fcn.py:12); `torchvision.models.vgg16` is replaced by a
    weights=None build before the constructor runs, so nothing is downloaded;
  * fcn.py:75-76 reads the undefined names `freeze_backbone` and `set_trainable` (every construction raises NameError
    without them); `freeze_backbone = False` and utils.helpers.set_trainable are injected into the module's globals;
  * dropout p = 0 for the train parity (the oracle does not model dropout).
Cases (21 classes, CrossEntropyLoss2d(ignore_index=255)), each a train step (loss, sampled logits, argmax, gradient norms,
selected gradients) followed by an eval forward:
  s64/     2x3x64x64: the padded input is 262 wide, every pool input is even
  s50x75/  2x3x50x75: pool input widths 273, 137, 69, 35, 18 and heights 248, 124, 62, 31, 16: partial ceil windows at the
           first four pools
"""
import os

import numpy as np
import torch

from .make_golden import OUT, import_reference, no_dropout

SMALL_GRADS = ["pool3.0.weight", "pool5.4.bias", "adj_pool3.weight", "adj_pool3.bias", "adj_pool4.bias", "output.6.bias"]
CASES = (("s64/", 64, 64, 31, 9031), ("s50x75/", 50, 75, 32, 9032))
NUM_CLASSES = 21


def install_vgg_shim():
    """torchvision.models.vgg16 -> the same network built with weights=None (fcn.py:12 calls it by attribute)."""
    import torchvision
    orig = torchvision.models.vgg16
    if getattr(orig, "_weights_none_shim", False):
        return

    def vgg16(*args, **kwargs):
        kwargs.pop("pretrained", None)
        args = ()
        kwargs["weights"] = None
        return orig(*args, **kwargs)

    vgg16._weights_none_shim = True
    torchvision.models.vgg16 = vgg16


def import_fcn():
    """models.fcn with the shims above applied (the reference tree must already be on sys.path)."""
    install_vgg_shim()
    import importlib
    from utils.helpers import set_trainable
    F = importlib.import_module("models.fcn")
    F.freeze_backbone = False
    F.set_trainable = set_trainable
    return F


def train_step(ref, sd, x, y, crit, prefix, rec):
    ref.load_state_dict(sd, strict=True)  # proves the oracle's key names and shapes are the reference's
    no_dropout(ref)
    ref.train()
    out = ref(x)
    loss = crit(out, y)
    loss.backward()
    params = dict(ref.named_parameters())
    rec[prefix + "param_names"] = np.array(list(params))
    rec[prefix + "grad_norms"] = np.array([0.0 if p.grad is None else p.grad.double().norm().item() for p in params.values()])
    rec[prefix + "loss"] = np.float64(loss.item())
    rec[prefix + "out_shape"] = np.array(out.shape)
    rec[prefix + "logits_sub"] = out.detach()[:, :, ::4, ::4].numpy()
    rec[prefix + "logits_sum"] = out.detach().double().sum((2, 3)).numpy()
    rec[prefix + "argmax"] = out.detach().argmax(1).to(torch.uint8).numpy()
    for n in SMALL_GRADS:
        rec[prefix + "grad/" + n] = params[n].grad.numpy()
    ref.eval()
    with torch.no_grad():
        rec[prefix + "eval_logits_sum"] = ref(x).double().sum((2, 3)).numpy()
    print(prefix, "loss", loss.item(), "out", tuple(out.shape), "params", len(params))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_num_threads(8)
    models, losses = import_reference()
    F = import_fcn()
    from oracle import fcn, synth

    rec = {}
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    for prefix, h, w, seed, xseed in CASES:
        sd = fcn.fcn8_state_dict(NUM_CLASSES, seed=seed)
        x, y = synth.make_batch(2, h, w, NUM_CLASSES, 255, seed=xseed)
        train_step(F.FCN8(NUM_CLASSES, pretrained=False), sd, x, y, crit, prefix, rec)
    np.savez_compressed(os.path.join(OUT, "fcn.npz"), **rec)
    print("fcn.npz written")


if __name__ == "__main__":
    main()
