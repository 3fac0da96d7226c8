"""Generate tests/golden/pspdensenet.npz by running the UNMODIFIED reference models/pspnet.py PSPDenseNet (densenet121,
pretrained=False: the custom block0, torchvision's trunk built with weights=None) on oracle-made weights and synthetic
inputs (build container only, like oracle/make_golden.py):

    python -m oracle.make_golden_pspdensenet

Dropout p = 0 for the train parity (the oracle does not model dropout).  Cases (21 classes, CrossEntropyLoss2d(ignore_index
=255) on the main head + 0.4 x on the aux head, trainer.py:57-60), each a train step (loss, sampled logits, argmax, gradient
norms, selected gradients, block0.4's running statistics after its two updates) followed by an eval forward:
  s64/     2x3x64x64: the stem gives 31x31, the pool input 14x14 — nothing is dropped
  s70x78/  2x3x70x78: the unpadded stride-2 stem drops a trailing row and column (34x38), and so does the floor-mode
           average pool (its input 15x17, pooled 7x8)
"""
import os

import numpy as np
import torch

from .make_golden import OUT, import_reference, no_dropout

BACKBONE = "densenet121"
NUM_CLASSES = 21
CASES = (("s64/", 64, 64, 41, 9041), ("s70x78/", 70, 78, 42, 9042))
# gradients recorded whole; block0.3.weight (the conv applied twice: the sum of both uses) by its first 8 output channels
SMALL_GRADS = ["block0.4.weight", "block0.4.bias", "transition3.0.bias", "master_branch.0.bottleneck.1.weight",
               "master_branch.1.bias", "auxiliary_branch.4.bias"]
SLICED_GRADS = {"block0.3.weight": 8, "master_branch.1.weight": 4}


def train_step(ref, sd, x, y, crit, prefix, rec):
    ref.load_state_dict(sd, strict=True)  # proves the oracle's key names and shapes are the reference's
    no_dropout(ref)
    ref.train()
    out, aux = ref(x)
    loss = crit(out, y) + 0.4 * crit(aux, y)
    loss.backward()
    params = dict(ref.named_parameters())
    rec[prefix + "param_names"] = np.array(list(params))
    rec[prefix + "grad_norms"] = np.array([0.0 if p.grad is None else p.grad.double().norm().item() for p in params.values()])
    rec[prefix + "loss"] = np.float64(loss.item())
    rec[prefix + "out_shape"] = np.array(out.shape)
    rec[prefix + "logits_sub"] = out.detach()[:, :, ::4, ::4].numpy()
    rec[prefix + "logits_sum"] = out.detach().double().sum((2, 3)).numpy()
    rec[prefix + "aux_sum"] = aux.detach().double().sum((2, 3)).numpy()
    rec[prefix + "argmax"] = out.detach().argmax(1).to(torch.uint8).numpy()
    for n in SMALL_GRADS:
        rec[prefix + "grad/" + n] = params[n].grad.numpy()
    for n, k in SLICED_GRADS.items():
        rec[prefix + "grad_head/" + n] = params[n].grad[:k].numpy()
    bsd = ref.state_dict()
    for n in ("block0.4.running_mean", "block0.4.running_var", "block0.4.num_batches_tracked"):
        rec[prefix + "buf/" + n] = bsd[n].numpy()
    ref.eval()
    with torch.no_grad():
        rec[prefix + "eval_logits_sum"] = ref(x).double().sum((2, 3)).numpy()
    print(prefix, "loss", loss.item(), "out", tuple(out.shape), "params", len(params))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    torch.set_num_threads(8)
    _, losses = import_reference()
    import importlib
    P = importlib.import_module("models.pspnet")
    from oracle import pspdensenet, synth

    rec = {}
    crit = losses.CrossEntropyLoss2d(ignore_index=255)
    for prefix, h, w, seed, xseed in CASES:
        sd = pspdensenet.pspdensenet_state_dict(NUM_CLASSES, BACKBONE, seed=seed)
        x, y = synth.make_batch(2, h, w, NUM_CLASSES, 255, seed=xseed)
        train_step(P.PSPDenseNet(NUM_CLASSES, backbone=BACKBONE, pretrained=False), sd, x, y, crit, prefix, rec)
    np.savez_compressed(os.path.join(OUT, "pspdensenet.npz"), **rec)
    print("pspdensenet.npz written")


if __name__ == "__main__":
    main()
