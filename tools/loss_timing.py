"""Times the per-pixel losses on the GPU with CUDA events: unweighted CE, class-weighted CE and focal loss (gamma 2, with
class weights), forward + backward, on both paths:
  * fused: bilinear upsample + loss from the low-resolution NHWC fp32 logits (seg_upsample_loss_*), as FusedTrainStep
    runs it;
  * nchw: the loss on full-resolution NCHW fp32 logits (seg_loss_nchw_*), as the plugin surface runs it.
Shapes: C3 (19 classes, 129x129 -> 513x513, batch 16) and C5 (150 classes, 128x128 -> 512x512, batch 8).

    python tools/loss_timing.py [--iters 50] [--rounds 5] [--out FILE]

Each round times every (loss, path) pair of a shape once, in turn, so that clock and neighbour drift spread over all of
them; the median over the rounds is reported.  Prints the device name and power limit with the numbers; there is no CPU
mode.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

SHAPES = {"C3": (16, 19, 129, 513, True, 255), "C5": (8, 150, 128, 512, False, -1)}


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - the numbers are still worth printing without it
        q = f"unavailable ({e})"
    return name, q


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_timing: needs a CUDA device")
    from seg_b200 import lib, ops
    lib.require_device()
    name, power = device_info()
    print(f"device: {name}; power.limit, clocks.max.sm: {power}")
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for shape, (N, C, Hi, Ho, ac, ign) in SHAPES.items():
        lo = torch.randn(N, Hi, Hi, C, device="cuda", generator=g) * 3
        target = torch.randint(0, C, (N, Ho, Ho), device="cuda", generator=g)
        target[:, :16] = ign
        w = torch.rand(C, device="cuda", generator=g) + 0.5
        ldx = (C + 7) // 8 * 8
        full = torch.randn(N, C, Ho, Ho, device="cuda", generator=g) * 3
        variants = {"ce": (None, None), "weighted_ce": (w, None), "focal_g2_weighted": (w, 2.0)}
        fns = {}
        for vname, v in variants.items():
            def fused(v=v):
                _, acc, _ = ops.upsample_loss_fwd(lo, target, ac, ign, v[0], v[1])
                ops.upsample_loss_bwd(lo, target, ac, ign, acc, ldx, v[0], v[1])

            def nchw(v=v):
                _, acc = ops.loss_nchw_fwd(full, target, ign, v[0], v[1])
                ops.loss_nchw_bwd(full, target, ign, acc, v[0], v[1])
            fns[("fused", vname)], fns[("nchw", vname)] = fused, nchw
        times = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, fn in fns.items():
                times[k].append(timed(fn, a.iters))
        for (path, vname), ts in sorted(times.items()):
            ms = statistics.median(ts)
            rows.append({"shape": shape, "loss": vname, "path": path, "ms_fwd_bwd": round(ms, 3),
                         "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3)})
            print(f"{shape} {path:5s} {vname:18s} fwd+bwd median {ms:8.3f} ms (range {min(ts):.3f}-{max(ts):.3f})")
        del full
        torch.cuda.empty_cache()
    for shape in SHAPES:
        for path in ("fused", "nchw"):
            base = next(r["ms_fwd_bwd"] for r in rows if r["shape"] == shape and r["path"] == path and r["loss"] == "ce")
            rel = ", ".join(f"{r['loss']} {r['ms_fwd_bwd'] / base:.3f}x" for r in rows
                            if r["shape"] == shape and r["path"] == path and r["loss"] != "ce")
            print(f"{shape} {path}: relative to CE: {rel}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"device": name, "power_limit_max_sm_clock": power, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
