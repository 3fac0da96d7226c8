"""Times one FCN8 training step on the GPU with CUDA events, at the configs' crop and batch: 8 x 3 x 512^2 and 8 x 3 x 513^2;
21 classes (and --classes 150), cross-entropy with ignore_index 255, SGD (lr 0.01, momentum 0.9, weight decay 1e-4, the
backbone group at lr / 10; base/base_trainer.py:46-57).

  fused      FusedTrainStep(model, cuda_graph=True).step(x, y)
  plugin     model.cuda_graphs(True); CrossEntropyLoss2d(model(x), y).backward(); torch.optim.SGD.step()  (trainer.py:55-71)
  reference  the unmodified models/fcn.py from oracle/_ref/reference.zip, fp32 NCHW, cuDNN with cudnn.benchmark,
             utils.losses.CrossEntropyLoss2d, torch.optim.SGD, built under the shim of oracle/make_golden_fcn.py:
             torchvision's vgg16 with weights=None, and the undefined `freeze_backbone` / `set_trainable` of fcn.py:75-76
             injected (without them the reference cannot be constructed)
  kernels    (--kernels) the new kernels per launch at the model's shapes: the ReLU + ceil pools (GB/s from the bytes they
             must move), conv6 / conv7's ReLU + dropout, and the three score upsamplers forward and data gradient (TFLOP/s
             from 2 * pixels * 4C * C, the padded-free algorithmic count)

    python tools/fcn_timing.py [--iters 5] [--rounds 5] [--legs fused,plugin,reference] [--sizes 512,513] [--classes 21,150]
                               [--kernels] [--out FILE]

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

N = 8


def sgd(model, lr=0.01):
    groups = [{"params": model.get_decoder_params()}, {"params": model.get_backbone_params(), "lr": lr * 0.1}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9, weight_decay=1e-4)


def fused_leg(C):
    import seg_b200
    from seg_b200.train import FusedTrainStep
    stepper = FusedTrainStep(seg_b200.FCN8(C, pretrained=False).cuda().train(), ignore_index=255, cuda_graph=True)
    return lambda x, y: stepper.step(x, y)


def plugin_leg(C):
    import seg_b200
    model = seg_b200.FCN8(C, pretrained=False).cuda().train().cuda_graphs(True, warmup=2)
    crit, opt = seg_b200.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def reference_leg(C):
    from bench import _import_reference_tree
    if _import_reference_tree() is None:
        raise SystemExit("fcn_timing: oracle/_ref/reference.zip not built (build() packs it from a reference checkout)")
    import importlib
    import torchvision
    vgg16 = torchvision.models.vgg16
    if not getattr(vgg16, "_weights_none", False):
        def shim(*args, **kwargs):
            kwargs.pop("pretrained", None)
            return vgg16(**{**kwargs, "weights": None})
        shim._weights_none = True
        torchvision.models.vgg16 = shim
    from utils import losses
    from utils.helpers import set_trainable
    Fm = importlib.import_module("models.fcn")
    Fm.freeze_backbone, Fm.set_trainable = False, set_trainable
    torch.backends.cudnn.benchmark = True
    model = Fm.FCN8(C, pretrained=False).cuda().train()
    crit, opt = losses.CrossEntropyLoss2d(ignore_index=255), sgd(model)

    def step(x, y):
        opt.zero_grad()
        crit(model(x), y).backward()
        opt.step()
    return step


def pool_sizes(S):
    """[(channels, H) of the map in front of each ceil-mode pool] and the class-map sizes (h, h2, h4) at an S x S input."""
    h, out = S + 198, []
    for c in (64, 128, 256, 512, 512):
        out.append((c, h))
        h = (h + 1) // 2
    h6 = h - 6
    return out, (h6, 2 * h6 + 2, 4 * h6 + 6)


def kernel_rows(S, C, iters):
    from seg_b200 import ops
    from seg_b200.nets import upsampling_weight
    rows = []

    def add(op, shape, fn, nbytes=None, flops=None):
        ms = statistics.median(timed(fn, iters) for _ in range(5))
        r = {"op": op, "shape": shape, "ms": round(ms, 4)}
        if nbytes:
            r["GB_per_s"] = round(nbytes / ms / 1e6, 1)
            r["share_of_3350"] = round(nbytes / ms / 1e6 / 3350.0, 3)
        if flops:
            r["TFLOP_per_s"] = round(flops / ms / 1e9, 1)
        rows.append(r)
        print(json.dumps(r))

    pools, (h6, h2, h4) = pool_sizes(S)
    for c, H in pools:
        x = torch.randn(N, H, H, c, device="cuda").bfloat16()
        y, code = ops.relu_maxpool2x2_ceil_fwd(x)
        dy = torch.randn_like(y)
        full, pooled = N * H * H * c, y.numel()
        add("relu_maxpool2x2_ceil_fwd", f"{N}x{H}x{H}x{c}", lambda: ops.relu_maxpool2x2_ceil_fwd(x), nbytes=2 * full + 3 * pooled)
        add("relu_maxpool2x2_ceil_bwd", f"{N}x{H}x{H}x{c}", lambda: ops.relu_maxpool2x2_ceil_bwd(dy, code, tuple(x.shape)),
            nbytes=3 * pooled + 2 * full)
    x = torch.randn(N * h6 * h6, 4096, device="cuda").bfloat16()
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    add("relu_dropout_fwd", f"{N * h6 * h6}x4096", lambda: ops.relu_dropout_fwd(x, 0.5, 1, ctr), nbytes=4 * x.numel())
    for name, k, hin, win in (("up_output", 4, h6, (0, 0, h2, h2)), ("up_pool4_out", 4, h2, (0, 0, h4, h4)),
                              ("up_final", 16, h4, (31, 31, S, S))):
        w = upsampling_weight(C, C, k).cuda()
        wf, wb = ops.score_pack(w, False), ops.score_pack(w, True)
        xin = torch.randn(N, hin, hin, (C + 7) // 8 * 8, device="cuda").bfloat16()[..., :C]
        dt = torch.float32 if name == "up_final" else torch.bfloat16
        y = ops.score_upsample_fwd(xin, wf, k, win, out_dtype=dt)
        dy = torch.randn(N, win[2], win[3], (C + 7) // 8 * 8, device="cuda").bfloat16()[..., :C]
        flops = 2.0 * N * win[2] * win[3] * 4 * C * C
        add(f"score_fwd {name}", f"{N}x{hin}^2 -> window {win[2]}^2, C={C}", lambda: ops.score_upsample_fwd(xin, wf, k, win, out_dtype=dt),
            flops=flops)
        add(f"score_bwd {name}", f"{N}x{hin}^2 <- window {win[2]}^2, C={C}",
            lambda: ops.score_upsample_bwd(dy, wb, tuple(xin.shape), k, win), flops=flops)
        del y
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--legs", default="fused,plugin,reference")
    ap.add_argument("--sizes", default="512,513")
    ap.add_argument("--classes", default="21")
    ap.add_argument("--kernels", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fcn_timing: needs a CUDA device")
    from seg_b200 import lib
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    sizes = [int(v) for v in a.sizes.split(",")]
    results = {"device": name, "power_limit_max_sm_clock": power, "batch": N, "sizes": sizes, "iters": a.iters,
               "rounds": a.rounds, "runs": []}
    for C in (int(v) for v in a.classes.split(",")):
        kernels = {S: kernel_rows(S, C, 20) for S in sizes} if a.kernels else {}
        legs = {}
        for leg in filter(None, a.legs.split(",")):
            torch.manual_seed(0)
            legs[leg] = {"fused": fused_leg, "plugin": plugin_leg, "reference": reference_leg}[leg](C)
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
            print(f"{C:3d} classes {k:10s} {N}x3x{S}x{S} median {ms:9.2f} ms/step (range {min(ts):.2f}-{max(ts):.2f}), "
                  f"{N * 1000.0 / ms:7.1f} img/s")
        results["runs"].append({"classes": C, "rows": rows, "kernels": kernels})
        del legs, batches
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
