"""Times one DeepLab_DUC_HDC training step on the GPU with CUDA events, at the configs' shape: 8 x 3 x 512^2, 19 classes,
cross-entropy with ignore_index 255, SGD (lr 0.01, backbone x 0.1, momentum 0.9, weight decay 1e-4; base/base_trainer.py:46-57).

  fused      FusedTrainStep(model, cuda_graph=True).step(x, y)
  plugin     model.cuda_graphs(True); CrossEntropyLoss2d(model(x), y).backward(); torch.optim.SGD.step()  (trainer.py:55-71)
  reference  the unmodified models/duc_hdc.py from oracle/_ref/reference.zip (its constructor needs the module globals
             freeze_backbone / set_trainable, duc_hdc.py:225), fp32 NCHW, cuDNN with cudnn.benchmark, utils.losses
             .CrossEntropyLoss2d, torch.optim.SGD

    python tools/duc_hdc_timing.py [--iters 5] [--rounds 5] [--legs fused,plugin,reference] [--out FILE]

Every leg is warmed up first; each round then times every leg once, in turn, so that clock and neighbour drift spread over all
of them; the median over the rounds is reported.  Prints the device name, power limit and max SM clock with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from loss_timing import device_info, timed  # noqa: E402

N, S, C = 8, 512, 19


def sgd(model, lr=0.01):
    groups = [{"params": model.get_decoder_params()}, {"params": model.get_backbone_params(), "lr": lr * 0.1}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9, weight_decay=1e-4)


def fused_leg():
    import seg_b200
    from seg_b200.train import FusedTrainStep
    stepper = FusedTrainStep(seg_b200.DeepLab_DUC_HDC(C, pretrained=False).cuda().train(), ignore_index=255, cuda_graph=True)
    return lambda x, y: stepper.step(x, y)


def plugin_leg():
    import seg_b200
    model = seg_b200.DeepLab_DUC_HDC(C, pretrained=False).cuda().train().cuda_graphs(True, warmup=2)
    crit, opt = seg_b200.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def reference_leg():
    from bench import _import_reference_tree
    if _import_reference_tree() is None:
        raise SystemExit("duc_hdc_timing: oracle/_ref/reference.zip not built (build() packs it from a reference checkout)")
    import models.duc_hdc as D
    from utils import helpers, losses
    D.freeze_backbone, D.set_trainable = False, helpers.set_trainable
    torch.backends.cudnn.benchmark = True
    model = D.DeepLab_DUC_HDC(C, pretrained=False).cuda().train()
    crit, opt = losses.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--legs", default="fused,plugin,reference")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("duc_hdc_timing: needs a CUDA device")
    from seg_b200 import lib
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, 3, S, S, device="cuda", generator=g)
    y = torch.randint(0, C, (N, S, S), device="cuda", generator=g)
    y[:, :16] = 255
    legs = {}
    for leg in a.legs.split(","):
        torch.manual_seed(0)
        legs[leg] = {"fused": fused_leg, "plugin": plugin_leg, "reference": reference_leg}[leg]()
        for _ in range(3):  # graph capture (fused / plugin), cudnn.benchmark's algorithm search (reference)
            legs[leg](x, y)
        torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(a.rounds):
        for k, fn in legs.items():
            times[k].append(timed(lambda: fn(x, y), a.iters))
    rows = []
    for k, ts in times.items():
        ms = statistics.median(ts)
        rows.append({"leg": k, "ms_per_step": round(ms, 2), "min_ms": round(min(ts), 2), "max_ms": round(max(ts), 2),
                     "img_per_s": round(N * 1000.0 / ms, 1)})
        print(f"{k:10s} median {ms:9.2f} ms/step (range {min(ts):.2f}-{max(ts):.2f}), {N * 1000.0 / ms:7.1f} img/s")
    res = {"device": name, "power_limit_max_sm_clock": power, "shape": [N, 3, S, S], "classes": C, "iters": a.iters,
           "rounds": a.rounds, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
