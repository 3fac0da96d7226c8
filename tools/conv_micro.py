#!/usr/bin/env python
"""Micro-benchmark of one convolution shape through the C ABI (for ncu captures and kernel tuning).

    python tools/conv_micro.py --shape 16,33,33,256,1024,1,1,1 --kind fwd --iters 50
    shape = N,H,W,C,K,ksize,stride,dil   (pad = dil*(ksize-1)/2);  kind in fwd|dgrad|wgrad|all
Prints CUDA-event time per launch, TFLOP/s and GB/s (algorithmic).  Inputs are rotated over several buffers so the
126 MB L2 does not hold the working set between launches.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-segmentation_b200"))
import torch  # noqa: E402
from seg_b200 import lib, ops  # noqa: E402


def run(shape, kind, iters, stats, impl, beta=0.0):
    N, H, W, C, K, ks, stride, dil = shape
    pad = dil * (ks - 1) // 2
    P = lib.conv_out_size(H, ks, stride, pad, dil)
    Q = lib.conv_out_size(W, ks, stride, pad, dil)
    nbuf = 4
    xs = [torch.randn(N, H, W, C, device="cuda").to(torch.bfloat16) for _ in range(nbuf)]
    dys = [torch.randn(N, P, Q, K, device="cuda").to(torch.bfloat16) for _ in range(nbuf)]
    w = torch.randn(K, C, ks, ks, device="cuda") / (C * ks * ks) ** 0.5
    wp = ops.pack_weight(w)
    out_ys = [torch.empty(N, P, Q, K, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]
    out_dxs = [torch.zeros(N, H, W, C, device="cuda", dtype=torch.bfloat16) for _ in range(nbuf)]  # rotated: cold in L2
    dwp = torch.zeros(ks * ks, K, C, device="cuda")
    st = torch.zeros(2 * K, dtype=torch.float64, device="cuda") if stats else None
    flops = 2.0 * N * P * Q * K * C * ks * ks
    byt = {"fwd": (N * H * W * C + N * P * Q * K) * 2, "dgrad": (N * H * W * C + N * P * Q * K) * 2, "wgrad": (N * H * W * C + N * P * Q * K) * 2}

    def one(k, i):
        if k == "fwd":
            ops.conv2d_fwd(xs[i % nbuf], wp, K, ks, ks, stride, pad, dil, out=out_ys[i % nbuf], stats=st, impl=impl)
        elif k == "dgrad":
            ops.conv2d_dgrad(dys[i % nbuf], wp, (N, H, W, C), ks, ks, stride, pad, dil, out=out_dxs[i % nbuf], impl=impl, beta=beta)
        else:
            ops.conv2d_wgrad(dys[i % nbuf], xs[i % nbuf], ks, ks, stride, pad, dil, out=dwp, impl=impl)

    for k in (["fwd", "dgrad", "wgrad"] if kind == "all" else [kind]):
        for i in range(5):
            one(k, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            one(k, i)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        print(f"{k:6s} shape={shape} stats={int(bool(stats))} beta={beta}: {us:8.2f} us  {flops / us / 1e6:8.1f} TFLOP/s  {byt[k] / us / 1e3:8.1f} GB/s")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", action="append", required=True)
    ap.add_argument("--kind", default="all")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--stats", type=int, default=1)
    ap.add_argument("--impl", type=int, default=0)
    ap.add_argument("--beta", type=float, default=0.0, help="dgrad: accumulate into the existing gradient")
    a = ap.parse_args()
    lib.require_device()
    for s in a.shape:
        run(tuple(int(v) for v in s.split(",")), a.kind, a.iters, a.stats, a.impl, a.beta)
