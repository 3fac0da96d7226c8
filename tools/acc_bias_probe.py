#!/usr/bin/env python
"""Does the wgmma fp32 accumulator round or truncate?  Positive bf16 operands, 1x1 conv = GEMM with growing
reduction length; the engine's fp32 output and cuBLAS's (bf16 operands, fp32 output) are compared with a float64
product of the same bf16 values: mean SIGNED relative error (a systematic shrink shows up as a negative mean that grows
with the reduction length) and the rms relative error.

    python tools/acc_bias_probe.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-segmentation_b200"))
import torch  # noqa: E402
from seg_b200 import lib, ops  # noqa: E402

lib.require_device()
torch.backends.cuda.matmul.allow_tf32 = False
g = torch.Generator().manual_seed(0)
for signed in (False, True):
    for Kdim in (64, 256, 2304, 18432):
        M, N = 4096, 128
        a = torch.rand(M, Kdim, generator=g) + 0.5
        b = torch.rand(N, Kdim, generator=g) + 0.5
        if signed:
            a, b = a - 1.0, b - 1.0
        a, b = a.to(torch.bfloat16), b.to(torch.bfloat16)
        ref = (a.double() @ b.double().t())
        x = a.cuda().reshape(1, 64, 64, Kdim).contiguous()
        wp = ops.pack_weight(b.float().cuda().reshape(N, Kdim, 1, 1))
        y = ops.conv2d_fwd(x, wp, N, 1, 1, out_dtype=torch.float32).reshape(M, N).double().cpu()
        try:
            yt = torch.mm(a.cuda(), b.cuda().t(), out_dtype=torch.float32).double().cpu()
        except Exception:
            yt = (a.cuda().float() @ b.cuda().float().t()).double().cpu()
        scale = ref.abs().mean()
        for name, v in (("wgmma (engine)", y), ("cuBLAS bf16->fp32", yt)):
            err = (v - ref) / scale
            print(f"signed={int(signed)} K={Kdim:6d} {name:18s}: mean signed rel err {err.mean().item():+.3e}  rms {err.pow(2).mean().sqrt().item():.3e}  (fp32 eps 6e-8)")
