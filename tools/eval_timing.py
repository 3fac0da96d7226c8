"""Times the validation batch and the metrics of the training step on the GPU with CUDA events.

(a) One validation batch, both graph-replayed:
      * plugin: model.eval()(x) (full-resolution fp32 NCHW logits), the loss on them, then ops.eval_metrics_nchw into
        device counters (no host copy) -- what Trainer._valid_epoch runs per batch through the plugin surface;
      * fused: FusedTrainStep(metrics=True, cuda_graph=True).evaluate(x, y).
    At C3 (DeepLabV3+/ResNet-101, 16 x 3 x 513^2, 19 classes, align_corners=True) and at C5's shapes (UperNet/ResNet-101,
    8 x 3 x 512^2, 150 classes, align_corners=False) with cross-entropy.
(b) The graph-replayed training step at C3 with metrics off and on.

    python tools/eval_timing.py [--iters 10] [--rounds 5] [--out FILE]

Each round times every variant of a part once, in turn, so that clock and neighbour drift spread over all of them; the
median over the rounds is reported.  Prints the device name and power limit with the numbers; there is no CPU mode.
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

# name: (arch, constructor kwargs, classes, image size, batch); the loss is cross-entropy with ignore_index 255
SHAPES = {"C3": ("DeepLab", dict(backbone="resnet101", output_stride=16), 19, 513, 16),
          "C5": ("UperNet", dict(backbone="resnet101"), 150, 512, 8)}


def batch(C, S, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, 3, S, S, device="cuda", generator=g)
    y = torch.randint(0, C, (N, S, S), device="cuda", generator=g)
    y[:, :16] = 255
    return x, y


def rounds(fns, iters, n_rounds):
    times = {k: [] for k in fns}
    for _ in range(n_rounds):
        for k, fn in fns.items():
            times[k].append(timed(fn, iters))
    return {k: (statistics.median(ts), min(ts), max(ts)) for k, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_timing: needs a CUDA device")
    import seg_b200
    from seg_b200 import lib, ops
    from seg_b200.train import FusedTrainStep
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    rows = []

    def report(part, shape, res):
        for k, (ms, lo, hi) in res.items():
            rows.append({"part": part, "shape": shape, "variant": k, "ms": round(ms, 3), "min_ms": round(lo, 3), "max_ms": round(hi, 3)})
            print(f"{part} {shape} {k:12s} median {ms:8.3f} ms (range {lo:.3f}-{hi:.3f})")

    # (a) validation batch
    for shape, (arch, kw, C, S, N) in SHAPES.items():
        torch.manual_seed(0)
        model = getattr(seg_b200, arch)(C, pretrained=False, **kw).cuda().eval()
        model.cuda_graphs(True, warmup=2)
        crit = seg_b200.CrossEntropyLoss2d(ignore_index=255)
        x, y = batch(C, S, N, 1)
        stepper = FusedTrainStep(model, ignore_index=255, metrics=True, cuda_graph=True)

        @torch.no_grad()
        def plugin():
            out = model(x)
            crit(out, y)
            ops.eval_metrics_nchw(out, y, C)

        def fused():
            stepper.evaluate(x, y)

        report("validation", shape, rounds({"plugin": plugin, "fused": fused}, a.iters, a.rounds))
        stepper.release_graph()
        model.release_graphs()
        del model, stepper
        torch.cuda.empty_cache()

    # (b) training step, metrics off / on
    arch, kw, C, S, N = SHAPES["C3"]
    x, y = batch(C, S, N, 2)
    steppers = {}
    for met in (False, True):
        torch.manual_seed(0)
        model = getattr(seg_b200, arch)(C, pretrained=False, **kw).cuda().train()
        steppers["metrics_on" if met else "metrics_off"] = FusedTrainStep(model, ignore_index=255, lr=0.01, backbone_lr_scale=0.1,
                                                                          momentum=0.9, weight_decay=1e-4, cuda_graph=True,
                                                                          metrics=met)
    res = rounds({k: (lambda s=s: s.step(x, y)) for k, s in steppers.items()}, a.iters, a.rounds)
    report("train_step", "C3", res)
    for s in steppers.values():
        s.release_graph()
    for shape in SHAPES:
        r = {row["variant"]: row["ms"] for row in rows if row["part"] == "validation" and row["shape"] == shape}
        print(f"validation {shape}: fused / plugin = {r['fused'] / r['plugin']:.3f}")
    r = {row["variant"]: row["ms"] for row in rows if row["part"] == "train_step"}
    print(f"train_step C3: metrics on / off = {r['metrics_on'] / r['metrics_off']:.4f}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"device": name, "power_limit_max_sm_clock": power, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
