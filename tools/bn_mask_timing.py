#!/usr/bin/env python
"""Per-launch timing of the BatchNorm backward passes with the ReLU mask read from the activation (A, bf16), from the
bit mask written by the forward apply (bits, 1/16 of the bytes) or recomputed from the conv output (recompute, BN -> ReLU
maps only), and of bn_apply_train with and without writing the mask, at the large maps of the C3 step
(DeepLabV3+/ResNet-101, 16 x 513^2).

    python tools/bn_mask_timing.py [--rounds 7] [--iters 40] [--json out.json]
Inputs are rotated (working set > L2), every variant is timed with CUDA events over `iters` launches, and the variants
take turns within each round; the median over rounds is reported, with the algorithmic bytes per element and GB/s
against the H100 SXM's 3.35 TB/s.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-segmentation_b200"))
import torch  # noqa: E402
from seg_b200 import lib, ops  # noqa: E402

HBM_GBS = 3350.0
# (name, N, H, W, C, residual): the residual-stream conv3 maps of layers 3, 1 and 2, a layer-1 conv1/conv2 map and the
# layer-4 output map without a residual
SHAPES = [("layer3.conv3", 16, 33, 33, 1024, True), ("layer1.conv3", 16, 129, 129, 256, True),
          ("layer2.conv3", 16, 65, 65, 512, True), ("layer1.conv1", 16, 129, 129, 64, False),
          ("layer4.x2048", 16, 33, 33, 2048, False)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "power limit unknown"
    return f"{name}, {q}"


def time_launches(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(iters)  # warm-up on the spare accumulator block
    torch.cuda.synchronize()
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def variants(N, H, W, C, res, iters):
    """{name: (launch(i), bytes per element)} for one shape."""
    M = N * H * W
    nbuf = max(2, int(300e6 // (M * C * 2 * 4)) + 1)
    g = torch.Generator(device="cuda").manual_seed(C)
    mk = lambda: torch.randn((N, H, W, C), device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
    xs, dys, rs = [mk() for _ in range(nbuf)], [mk() for _ in range(nbuf)], [mk() for _ in range(nbuf)]
    outs = [torch.empty_like(xs[0]) for _ in range(nbuf)]
    dxs = [torch.empty_like(xs[0]) for _ in range(nbuf)]
    masks = [ops.relu_mask(xs[0]) for _ in range(nbuf)]
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    stats = [ops.bn_stats(x) for x in xs]
    saves = []
    for b in range(nbuf):
        _, s = ops.bn_apply_train(xs[b], stats[b], M, gamma, beta, 1e-5, 0.1, 0, None, None, res=rs[b] if res else None,
                                  out=outs[b], mask=masks[b])
        saves.append(s)
    sums = ops.bn_bwd_reduce(dys[0], outs[0], xs[0], saves[0], relu=True)
    nw = ops.bn_bwd_reduce_acc_words(C)
    acc = torch.zeros(nw * (iters + 1), dtype=torch.float64, device="cuda")  # zeroed accumulators, one block per launch

    def fwd(use_mask):
        return lambda i: ops.bn_apply_train(xs[i % nbuf], stats[i % nbuf], M, gamma, beta, 1e-5, 0.1, 0, None, None,
                                            res=rs[i % nbuf] if res else None, out=outs[i % nbuf],
                                            mask=masks[i % nbuf] if use_mask else None)

    def red(src):
        def f(i):
            b = i % nbuf
            ops.bn_bwd_reduce(dys[b], outs[b] if src == "A" else None, xs[b], saves[b], relu=True,
                              acc=acc[i * nw:(i + 1) * nw], gamma=gamma, beta=beta,
                              mask=masks[b] if src == "bits" else None)
        return f

    def app(src):
        def f(i):
            b = i % nbuf
            ops.bn_bwd_apply(dys[b], outs[b] if src == "A" else None, xs[b], saves[b], gamma, sums, M, relu=True, dx=dxs[b],
                             dres=rs[b] if res else None, beta=beta, mask=masks[b] if src == "bits" else None)
        return f

    mask_b = 1.0 / 8  # one bit per element
    dres_b = 2.0 if res else 0.0
    v = {"bn_apply_train": (fwd(False), 4.0 + dres_b), "bn_apply_train+mask": (fwd(True), 4.0 + dres_b + mask_b),
         "bn_bwd_reduce[A]": (red("A"), 6.0), "bn_bwd_reduce[bits]": (red("bits"), 4.0 + mask_b),
         "bn_bwd_apply[A]": (app("A"), 8.0 + dres_b), "bn_bwd_apply[bits]": (app("bits"), 6.0 + dres_b + mask_b)}
    if not res:  # BN -> ReLU with nothing in between: the mask can also be recomputed from x
        v["bn_bwd_reduce[recompute]"] = (red("recompute"), 4.0)
        v["bn_bwd_apply[recompute]"] = (app("recompute"), 6.0 + dres_b)
    return v, acc, M * C


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lib.require_device()
    gpu = card()
    print(f"# {gpu}")
    rows = []
    for name, N, H, W, C, res in SHAPES:
        v, acc, elems = variants(N, H, W, C, res, a.iters)
        times = {k: [] for k in v}
        for _ in range(a.rounds):
            for k, (fn, _) in v.items():  # variants take turns within each round
                acc.zero_()
                times[k].append(time_launches(fn, a.iters))
        for k, (_, bpe) in v.items():
            us = statistics.median(times[k])
            gbs = bpe * elems / us / 1e3
            rows.append(dict(shape=name, N=N, H=H, W=W, C=C, res=res, kernel=k, us=us, us_min=min(times[k]),
                             us_max=max(times[k]), bytes_per_elem=bpe, GBps=gbs, hbm_frac=gbs / HBM_GBS))
            print(f"{name:13s} {N}x{H}x{W}x{C:<5d} {k:26s} {us:8.1f} us  [{min(times[k]):7.1f}, {max(times[k]):7.1f}]  "
                  f"{bpe:6.3f} B/elem  {gbs:7.0f} GB/s  {100 * gbs / HBM_GBS:5.1f}% of {HBM_GBS:.0f}")
        del v, acc
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, rounds=a.rounds, iters=a.iters, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
