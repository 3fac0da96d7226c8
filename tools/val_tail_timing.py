#!/usr/bin/env python
"""Throughput of the validation tail and cost of the Gaussian blur in the training tail.

    python tools/val_tail_timing.py [--gpu] [--cpu] [--batch 8] [--rounds 7] [--iters 20] [--workers 4] [--json out.json]

--gpu: on synthetic 1024 x 2048 Cityscapes-sized frames (uint8 image, int32 label), crop 480 (the shipped config.json's
  val_loader), the device validation tail per batch
    * end to end: DeviceBatcher.stage_val (pack into pinned memory, one H2D copy, one kernel) up to a device synchronise;
    * kernel only: seg_augment_val_batch_u8 on the staged arena, CUDA events over `iters` launches;
  and the training tail at the shipped train_loader geometry (base_size 400 scale draws, rotate on, crop 380) with every
  sample blurred (k = 3) vs unblurred: seg_augment_full_blur_batch_u8 vs seg_augment_full_batch_u8 on the same arena,
  alternating within each round.  Medians over rounds; the card's name and power limit are printed with the numbers.
--cpu: the reference's per-sample CPU work for the same frames (_val_augmentation's cv2.resize + PIL NEAREST resize +
  centre crop, then np.uint8, ToTensor, Normalize, label -> int64, as base/base_dataset.py runs it), in one process and
  in `workers` processes (the config's val_loader uses 4), with the host's core count."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-segmentation_b200"))

MEAN, STD = [0.28689529, 0.32513294, 0.28389176], [0.17613647, 0.18099176, 0.17772235]
H, W, VAL_CROP, CROP, BASE = 1024, 2048, 480, 380, 400


def frames(n, seed=0):
    rs = np.random.RandomState(seed)
    return [(rs.randint(0, 256, (H, W, 3)).astype(np.uint8), rs.randint(-1, 34, (H, W)).astype(np.int32)) for _ in range(n)]


# ------------------------------------------------------------------------------------------------ CPU reference
def reference_val_sample(image, label, crop=VAL_CROP):
    """The reference's work per validation sample, the same library calls in the same order."""
    import cv2
    import torch
    from PIL import Image
    from torchvision import transforms
    image = image.astype(np.float32)  # the loaders hand float32 images on
    h, w = label.shape
    h, w = (crop, int(crop * w / h)) if h < w else (int(crop * h / w), crop)
    image = cv2.resize(image, (w, h), interpolation=cv2.INTER_LINEAR)
    label = np.asarray(Image.fromarray(label).resize((w, h), resample=Image.NEAREST), dtype=np.int32)
    h, w = label.shape
    sh, sw = (h - crop) // 2, (w - crop) // 2
    image, label = image[sh:sh + crop, sw:sw + crop], label[sh:sh + crop, sw:sw + crop]
    label = torch.from_numpy(np.array(label, dtype=np.int32)).long()
    image = Image.fromarray(np.uint8(image))
    return transforms.Normalize(MEAN, STD)(transforms.ToTensor()(image)), label


def _cpu_worker(args):
    import cv2
    import torch
    cv2.setNumThreads(0)  # as BaseDataSet.__init__ does
    torch.set_num_threads(1)  # as torch.utils.data.DataLoader does in its workers
    n, seed = args
    fr = frames(2, seed)
    t0 = time.perf_counter()
    for i in range(n):
        reference_val_sample(*fr[i % 2])
    return n, time.perf_counter() - t0


def cpu_rates(n, workers):
    import multiprocessing as mp
    _cpu_worker((2, 0))  # imports, first-call costs
    k, t = _cpu_worker((n, 1))
    one = k / t
    ctx = mp.get_context("spawn")
    with ctx.Pool(workers) as pool:
        pool.map(_cpu_worker, [(2, s) for s in range(workers)])
        t0 = time.perf_counter()
        res = pool.map(_cpu_worker, [(n, s) for s in range(workers)])
        wall = time.perf_counter() - t0
    return {"cpu_cores": os.cpu_count(), "cpu_one_process_img_s": one, "cpu_workers": workers,
            "cpu_workers_img_s": sum(r[0] for r in res) / wall}


# ------------------------------------------------------------------------------------------------ device
def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "power limit unknown"
    return f"{name}, {q}"


def event_us(fn, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def gpu_rates(B, rounds, iters):
    import random

    import torch
    from seg_b200 import lib, ops
    from seg_b200.data import DeviceBatcher, draw_crop_flip, draw_rotate, draw_scale, gaussian_taps

    lib.require_device()
    fr = frames(B, 1)
    b = DeviceBatcher(MEAN, STD, VAL_CROP, "cuda:0", max_bytes=B * H * W * 8 + (8 << 20))
    for _ in range(3):
        b.stage_val(fr)
    torch.cuda.synchronize()
    e2e, kern = [], []
    for _ in range(rounds):
        t0 = time.perf_counter()
        for _ in range(iters // 4 + 1):
            b.stage_val(fr)
        torch.cuda.synchronize()
        e2e.append((time.perf_counter() - t0) * 1e6 / (iters // 4 + 1))
    # kernel only, on an arena staged by stage_val (the last staged copy is the one in use)
    import seg_b200.data as sd
    captured = {}
    real = ops.augment_val_batch_u8

    def grab(arena, table, *a, **k):
        captured["args"] = (arena, table) + a
        captured["kw"] = k
        return real(arena, table, *a, **k)

    sd.ops.augment_val_batch_u8 = grab
    try:
        b.stage_val(fr)
    finally:
        sd.ops.augment_val_batch_u8 = real
    torch.cuda.synchronize()
    for _ in range(rounds):
        kern.append(event_us(lambda: real(*captured["args"], **captured["kw"]), iters))
    out = {"card": card(), "batch": B, "frame": f"{H}x{W}", "val_crop": VAL_CROP,
           "val_end_to_end_us_per_batch": statistics.median(e2e), "val_kernel_us_per_batch": statistics.median(kern)}
    out["val_end_to_end_img_s"] = B / out["val_end_to_end_us_per_batch"] * 1e6
    out["val_kernel_img_s"] = B / out["val_kernel_us_per_batch"] * 1e6

    # training tail at the shipped train_loader geometry, every sample blurred vs none
    random.seed(3)
    samples = []
    for im, lb in fr:
        h, w = draw_scale(H, W, BASE, scale=True)
        angle = draw_rotate(True)
        y0, x0, flip = draw_crop_flip(h, w, CROP, flip=True)
        samples.append((im, lb, h, w, angle, y0, x0, flip))
    bt = DeviceBatcher(MEAN, STD, CROP, "cuda:0", max_bytes=B * H * W * 8 + (8 << 20))
    real_full = ops.augment_full_batch_u8

    def grab_full(arena, table, *a, **k):
        captured["full"] = (arena, table) + a
        captured["fkw"] = k
        return real_full(arena, table, *a, **k)

    sd.ops.augment_full_batch_u8 = grab_full
    try:
        bt.stage_full(samples)
    finally:
        sd.ops.augment_full_batch_u8 = real_full
    arena, table = captured["full"][:2]
    taps = torch.tensor([gaussian_taps(0.8)] * B, dtype=torch.float32, device="cuda:0")
    blur = lambda: ops.augment_full_blur_batch_u8(arena, table, taps, *captured["full"][2:], **captured["fkw"])  # noqa: E731
    plain = lambda: real_full(*captured["full"], **captured["fkw"])  # noqa: E731
    xb, yb = blur()
    xp, yp = plain()
    assert torch.equal(yb, yp)
    for f in (blur, plain):
        event_us(f, 3)
    tb, tp = [], []
    for _ in range(rounds):
        tb.append(event_us(blur, iters))
        tp.append(event_us(plain, iters))
    out.update({"train_crop": CROP, "train_sizes": [s[2:4] for s in samples], "train_full_us_per_batch": statistics.median(tp),
                "train_full_blur_us_per_batch": statistics.median(tb)})
    out["blur_cost_us_per_batch"] = out["train_full_blur_us_per_batch"] - out["train_full_us_per_batch"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--cpu-samples", type=int, default=24)
    ap.add_argument("--json")
    a = ap.parse_args()
    res = {}
    if a.gpu:
        res.update(gpu_rates(a.batch, a.rounds, a.iters))
    if a.cpu:
        res.update(cpu_rates(a.cpu_samples, a.workers))
    for k, v in res.items():
        print(f"{k}: {v:.1f}" if isinstance(v, float) else f"{k}: {v}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
