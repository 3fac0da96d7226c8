#!/usr/bin/env python
"""Cost of the input pipeline per sample, reference vs the `dataloaders` / `base` overlays, at config.json's settings.

    python tools/loader_timing.py [--gpu] [--frames 16] [--batches 12] [--json out.json]

Builds a seeded synthetic Cityscapes tree of 1024 x 2048 frames in a temporary directory (smooth random RGB PNGs and
labelIds PNGs; their compression differs from real frames) and runs, against the unmodified reference packed by build()
into oracle/_ref/reference.zip:
  * CPU, one thread, per sample: the reference's CityScapesDataset.__getitem__ at the shipped train_loader settings
    (base_size 400, scale, rotate, flip, crop 380) and the overlay dataset's __getitem__ (decode + draws) plus its share
    of device_collate (the packing), both as the loader's workers run them;
  * H2D bytes per batch of 8, computed: the reference's fp32 image + int64 label batch, and the packed arena;
  * --gpu: img/s through the overlay DataPrefetcher over the overlay loader with the config's 8 workers (host clock around
    `batches` batches, each ending in a device synchronise), and the kernel time per batch (CUDA events around the
    augmentation kernel on a staged arena), with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pytorch-segmentation_b200")
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
H, W, B = 1024, 2048, 8
TRAIN = dict(batch_size=B, base_size=400, crop_size=380, augment=True, shuffle=True, scale=True, flip=True, rotate=True, blur=False,
             split="train", num_workers=8)


def make_tree(root, n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    di = os.path.join(root, "leftImg8bit_trainvaltest", "leftImg8bit", "train", "city0")
    dl = os.path.join(root, "gtFine_trainvaltest", "gtFine", "train", "city0")
    os.makedirs(di)
    os.makedirs(dl)
    for k in range(n):
        small = rng.integers(0, 256, (H // 16, W // 16, 3)).astype(np.uint8)
        img = np.asarray(Image.fromarray(small).resize((W, H), Image.BILINEAR))
        Image.fromarray(img).save(os.path.join(di, f"city0_{k:06d}_000019_leftImg8bit.png"))
        lab = np.asarray(Image.fromarray(rng.integers(0, 34, (H // 32, W // 32)).astype(np.uint8)).resize((W, H), Image.NEAREST))
        Image.fromarray(lab, mode="L").save(os.path.join(dl, f"city0_{k:06d}_000019_gtFine_labelIds.png"))


def inner(args):
    import random
    import torch
    from seg_b200 import launch
    launch.setup_paths(os.getcwd())
    torch.set_num_threads(1)
    import cv2
    cv2.setNumThreads(0)
    import importlib.util
    spec = importlib.util.spec_from_file_location("_ref_cityscapes", os.path.join(os.getcwd(), "dataloaders", "cityscapes.py"))
    refmod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(refmod)
    import dataloaders
    from seg_b200.data import device_collate
    res = {"frames": args.frames, "frame": [H, W], "batch": B}
    ref = refmod.CityScapes(data_dir=args.data, **TRAIN)
    ov = dataloaders.CityScapes(data_dir=args.data, **TRAIN)
    assert ov.dataset.device_mode

    def per_sample(ds):
        random.seed(0)
        ds[0]
        t = time.perf_counter()
        items = [ds[i] for i in range(len(ds))]
        return (time.perf_counter() - t) * 1e3 / len(ds), items

    res["cpu_ms_reference_getitem"], _ = per_sample(ref.dataset)
    ms, items = per_sample(ov.dataset)
    t = time.perf_counter()
    packed = [device_collate(items[i:i + B]) for i in range(0, len(items) - B + 1, B)]
    res["cpu_ms_overlay_getitem"] = ms
    res["cpu_ms_overlay_pack"] = (time.perf_counter() - t) * 1e3 / (len(packed) * B)
    res["cpu_ms_overlay_total"] = res["cpu_ms_overlay_getitem"] + res["cpu_ms_overlay_pack"]
    c = TRAIN["crop_size"]
    res["h2d_bytes_reference"] = B * 3 * c * c * 4 + B * c * c * 8
    res["h2d_bytes_overlay"] = int(np.mean([p.arena.numel() for p in packed]))
    res["cpu_threads"] = os.cpu_count()
    if args.gpu:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        res["gpu"] = q.stdout.strip()
        import base
        dev = torch.device("cuda:0")
        from seg_b200.data import launch_packed
        pb = packed[0].pin_memory()
        arena = pb.arena.to(dev)
        for _ in range(5):
            launch_packed(pb, arena, ov.MEAN, ov.STD)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            launch_packed(pb, arena, ov.MEAN, ov.STD)
        e1.record()
        torch.cuda.synchronize()
        res["kernel_ms_per_batch"] = e0.elapsed_time(e1) / 50
        res["kernel"] = pb.kind
        torch.manual_seed(0)
        pf = base.DataPrefetcher(ov, device=dev)
        n, t = 0, None
        for k, (x, y) in enumerate(pf):
            torch.cuda.synchronize()
            if k == 1:   # the first batch waits for the workers to start
                t, n = time.perf_counter(), 0
            elif k > 1:
                n += x.shape[0]
        res["prefetcher_img_per_s"] = n / (time.perf_counter() - t) if n else float("nan")
        res["prefetcher_batches"] = len(pf)
    print("RESULT " + json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--json", default=None)
    ap.add_argument("--inner", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--data", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.inner:
        return inner(args)
    if not os.path.isfile(REF_ZIP):
        sys.exit("loader_timing: oracle/_ref/reference.zip not built (build() found no reference checkout)")
    with tempfile.TemporaryDirectory() as d:
        ref = os.path.join(d, "reference")
        with zipfile.ZipFile(REF_ZIP) as z:
            z.extractall(ref)
        data = os.path.join(d, "cityscapes")
        make_tree(data, args.frames)
        env = dict(os.environ, PYTHONPATH=PKG)
        env.pop("SEG_DEVICE_DATA", None)
        cmd = [sys.executable, "-W", "ignore", os.path.abspath(__file__), "--inner", "--data", data, "--frames", str(args.frames)]
        r = subprocess.run(cmd + (["--gpu"] if args.gpu else []), env=env, cwd=ref, capture_output=True, text=True)
        line = [x for x in r.stdout.splitlines() if x.startswith("RESULT ")]
        if r.returncode != 0 or not line:
            sys.exit(r.stdout[-3000:] + r.stderr[-4000:])
        res = json.loads(line[-1][7:])
    for k, v in res.items():
        print(f"{k:28s} {v:.2f}" if isinstance(v, float) else f"{k:28s} {v}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
