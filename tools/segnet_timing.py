"""Times one SegNet training step on the GPU with CUDA events, at the configs' crop and batch: 8 x 3 x 512^2, and at
8 x 3 x 513^2 (the first pool drops a row and a column); 19 classes, cross-entropy with ignore_index 255, SGD (lr 0.01,
momentum 0.9, weight decay 1e-4; base/base_trainer.py:46-57; SegNet has no backbone group).

  fused      FusedTrainStep(model, cuda_graph=True).step(x, y)
  plugin     model.cuda_graphs(True); CrossEntropyLoss2d(model(x), y).backward(); torch.optim.SGD.step()  (trainer.py:55-71)
  reference  the unmodified models/segnet.py from oracle/_ref/reference.zip, fp32 NCHW, cuDNN with cudnn.benchmark,
             utils.losses.CrossEntropyLoss2d, torch.optim.SGD; torchvision's vgg16_bn is built with weights=None (the
             reference constructor always asks for ImageNet weights, segnet.py:16)
  kernels    (--kernels) the four 2x2 pooling kernels at SegNet's pool shapes for the batch (64 x 512^2, 128 x 256^2,
             256 x 128^2, 512 x 64^2, 512 x 32^2 at 512): time per launch and achieved GB/s from the bytes the op must move
             (bf16 values, one uint8 code per pooled element), against the H100 SXM's 3.35 TB/s of HBM3

    python tools/segnet_timing.py [--iters 5] [--rounds 5] [--legs fused,plugin,reference] [--sizes 512,513] [--kernels] [--out FILE]

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
    stepper = FusedTrainStep(seg_b200.SegNet(C, pretrained=False).cuda().train(), ignore_index=255, cuda_graph=True)
    return lambda x, y: stepper.step(x, y)


def plugin_leg():
    import seg_b200
    model = seg_b200.SegNet(C, pretrained=False).cuda().train().cuda_graphs(True, warmup=2)
    crit, opt = seg_b200.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def reference_leg():
    from bench import _import_reference_tree
    if _import_reference_tree() is None:
        raise SystemExit("segnet_timing: oracle/_ref/reference.zip not built (build() packs it from a reference checkout)")
    import torchvision
    vgg16_bn = torchvision.models.vgg16_bn
    torchvision.models.vgg16_bn = lambda *args, **kwargs: vgg16_bn(*args, **{**kwargs, "weights": None})
    import models.segnet as S
    from utils import losses
    torch.backends.cudnn.benchmark = True
    model = S.SegNet(C, pretrained=False).cuda().train()
    crit, opt = losses.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


POOL_SHAPES = ((64, 1), (128, 2), (256, 4), (512, 8), (512, 16))  # (channels, input size divisor) of each encoder pool


def kernel_rows(S, iters):
    """The four pooling kernels at the pool shapes of an N x 3 x S^2 batch: [(op, shape, ms, GB/s, share of 3.35 TB/s)]."""
    from seg_b200 import ops
    rows = []
    for Cc, div in POOL_SHAPES:
        H = W = S // div  # floor mode: the encoder map in front of each pool
        P, Q = H // 2, W // 2
        x = torch.randn(N, H, W, Cc, device="cuda").bfloat16()
        y, code = ops.maxpool2x2_fwd(x)
        dy = torch.randn_like(y)
        dyu = torch.randn_like(x)
        full, pooled = N * H * W * Cc, N * P * Q * Cc
        cases = (("maxpool2x2_fwd", lambda: ops.maxpool2x2_fwd(x), 2 * full + 3 * pooled),
                 ("maxpool2x2_bwd", lambda: ops.maxpool2x2_bwd(dy, code, tuple(x.shape)), 3 * pooled + 2 * full),
                 ("maxunpool2x2_fwd", lambda: ops.maxunpool2x2_fwd(y, code, (H, W)), 3 * pooled + 2 * full),
                 ("maxunpool2x2_bwd", lambda: ops.maxunpool2x2_bwd(dyu, code), 2 * full + 3 * pooled))
        for op, fn, nbytes in cases:
            ms = statistics.median(timed(fn, iters) for _ in range(5))
            gbs = nbytes / ms / 1e6
            rows.append({"op": op, "shape": f"{N}x{H}x{W}x{Cc}", "ms": round(ms, 4), "GB_per_s": round(gbs, 1),
                         "share_of_3350": round(gbs / 3350.0, 3)})
            print(f"{op:17s} {N}x{H}x{W}x{Cc:<4d} {ms * 1000:8.1f} us  {gbs:7.1f} GB/s  ({gbs / 3350.0:.0%} of 3.35 TB/s)")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--legs", default="fused,plugin,reference")
    ap.add_argument("--sizes", default="512,513")
    ap.add_argument("--kernels", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("segnet_timing: needs a CUDA device")
    from seg_b200 import lib
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    sizes = [int(v) for v in a.sizes.split(",")]
    kernels = {S: kernel_rows(S, 20) for S in sizes} if a.kernels else {}
    legs = {}
    for leg in filter(None, a.legs.split(",")):
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
           "rounds": a.rounds, "rows": rows, "kernels": kernels}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
