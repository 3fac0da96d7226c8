"""Times one UNetResnet (resnet50) training step on the GPU with CUDA events, at the configs' crop and batch: 8 x 3 x 512^2,
and at 8 x 3 x 513^2 (every resample path of the decoder runs); 19 classes, cross-entropy with ignore_index 255, SGD (lr 0.01,
backbone x 0.1, momentum 0.9, weight decay 1e-4; base/base_trainer.py:46-57).

  fused      FusedTrainStep(model, cuda_graph=True).step(x, y)
  plugin     model.cuda_graphs(True); CrossEntropyLoss2d(model(x), y).backward(); torch.optim.SGD.step()  (trainer.py:55-71)
  reference  the unmodified models/unet.py from oracle/_ref/reference.zip, fp32 NCHW, cuDNN with cudnn.benchmark (its
             ConvTranspose2d included), utils.losses.CrossEntropyLoss2d, torch.optim.SGD

    python tools/unet_resnet_timing.py [--iters 5] [--rounds 5] [--legs fused,plugin,reference] [--sizes 512,513] [--out FILE]

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

N, C = 8, 19


def sgd(model, lr=0.01):
    groups = [{"params": model.get_decoder_params()}, {"params": model.get_backbone_params(), "lr": lr * 0.1}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9, weight_decay=1e-4)


def fused_leg():
    import seg_b200
    from seg_b200.train import FusedTrainStep
    stepper = FusedTrainStep(seg_b200.UNetResnet(C, pretrained=False).cuda().train(), ignore_index=255, cuda_graph=True)
    return lambda x, y: stepper.step(x, y)


def plugin_leg():
    import seg_b200
    model = seg_b200.UNetResnet(C, pretrained=False).cuda().train().cuda_graphs(True, warmup=2)
    crit, opt = seg_b200.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def reference_leg():
    from bench import _import_reference_tree
    if _import_reference_tree() is None:
        raise SystemExit("unet_resnet_timing: oracle/_ref/reference.zip not built (build() packs it from a reference checkout)")
    import models.unet as U
    from utils import losses
    torch.backends.cudnn.benchmark = True
    model = U.UNetResnet(C, backbone="resnet50", pretrained=False).cuda().train()
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
    ap.add_argument("--sizes", default="512,513")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unet_resnet_timing: needs a CUDA device")
    from seg_b200 import lib
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    sizes = [int(v) for v in a.sizes.split(",")]
    legs = {}
    for leg in a.legs.split(","):
        torch.manual_seed(0)
        legs[leg] = {"fused": fused_leg, "plugin": plugin_leg, "reference": reference_leg}[leg]()
    batches = {}
    for S in sizes:
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(N, 3, S, S, device="cuda", generator=g)
        y = torch.randint(0, C, (N, S, S), device="cuda", generator=g)
        y[:, :16] = 255
        batches[S] = (x, y)
        for fn in legs.values():
            for _ in range(3):  # graph capture (fused / plugin), cudnn.benchmark's algorithm search (reference)
                fn(x, y)
        torch.cuda.synchronize()
    times = {(k, S): [] for S in sizes for k in legs}
    for _ in range(a.rounds):
        for (k, S) in times:
            x, y = batches[S]
            times[(k, S)].append(timed(lambda: legs[k](x, y), a.iters))
    rows = []
    for (k, S), ts in times.items():
        ms = statistics.median(ts)
        rows.append({"leg": k, "size": S, "ms_per_step": round(ms, 2), "min_ms": round(min(ts), 2), "max_ms": round(max(ts), 2),
                     "img_per_s": round(N * 1000.0 / ms, 1)})
        print(f"{k:10s} {N}x3x{S}x{S} median {ms:9.2f} ms/step (range {min(ts):.2f}-{max(ts):.2f}), {N * 1000.0 / ms:7.1f} img/s")
    res = {"device": name, "power_limit_max_sm_clock": power, "batch": N, "sizes": sizes, "classes": C, "iters": a.iters,
           "rounds": a.rounds, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
