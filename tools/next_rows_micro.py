#!/usr/bin/env python
"""Measurement of the §8(f) "next" rows on one H100 (CUDA events, warm-up, synchronised on both sides):

  * input-pipeline tail: `seg_augment_batch_u8` achieved GB/s (algorithmic bytes: uint8 image + label read once, fp32
    image + int64 label written once) next to the reference's CPU tail (oracle/data.py restatement) on the host cores;
  * test-time augmentation: `seg_b200.inference.multi_scale_predict` / `sliding_predict` around the engine model, next to
    the reference's host-round-trip algorithm (oracle/inference.py restatement: ndimage.zoom + CPU up-sampling + numpy
    accumulation) around the SAME engine model;
  * `seg_b200.optim.SGD.step` vs `torch.optim.SGD.step` on the DeepLab-R101 parameter set.

    python tools/next_rows_micro.py > gpurun_out/next_rows.txt
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-segmentation_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import seg_b200  # noqa: E402
from seg_b200 import inference as di  # noqa: E402
from seg_b200.data import DeviceBatcher  # noqa: E402
from seg_b200.optim import SGD as FusedSGD  # noqa: E402
from oracle import data as od  # noqa: E402
from oracle import inference as oi  # noqa: E402


def ev_time(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    only = sys.argv[sys.argv.index("--only") + 1] if "--only" in sys.argv else None  # "tail": stop after the input-pipeline section
    torch.cuda.set_device(0)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    peak = 6580.0
    try:
        import json
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    rs = np.random.RandomState(0)
    # ---------------------------------------------------------------- input-pipeline tail
    B, crop = 16, 513
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    samples = []
    for _ in range(B):
        h, w = int(rs.randint(520, 900)), int(rs.randint(520, 1100))
        samples.append((rs.randint(0, 256, (h, w, 3)).astype(np.uint8), rs.randint(0, 21, (h, w)).astype(np.uint8),
                        int(rs.randint(0, h - crop + 1)), int(rs.randint(0, w - crop + 1)), bool(rs.rand() > 0.5)))
    b = DeviceBatcher(mean, std, crop, "cuda:0", max_bytes=128 << 20)
    x, y = b.stage(samples)  # warm
    torch.cuda.synchronize()
    # kernel alone: arena already on the device
    from seg_b200 import ops
    host = b._host[b._slot ^ 1]
    dev = host[:b.last_staged_bytes].cuda()
    tab = dev[:B * 40]
    ms = ev_time(lambda: ops.augment_batch_u8(dev, tab, B, crop, crop, mean, std), 50)
    alg = B * crop * crop * (3 + 1 + 12 + 8)
    print(f"[tail] seg_augment_batch_u8 B={B} crop={crop}: {ms * 1e3:.1f} us/launch, algorithmic {alg / 1e6:.1f} MB -> "
          f"{alg / (ms * 1e-3) / 1e9:.0f} GB/s = {alg / (ms * 1e-3) / 1e9 / peak:.2f} of the measured HBM peak ({peak:.0f} GB/s)")
    ms_stage = ev_time(lambda: b.stage(samples), 10)
    h2d = sum(s[0].size + s[1].size for s in samples)
    print(f"[tail] DeviceBatcher.stage (host pack + H2D of {h2d / 1e6:.1f} MB uint8 + kernel): {ms_stage:.2f} ms/batch "
          f"({B / ms_stage * 1e3:.0f} img/s on one host thread); the reference ships {B * crop * crop * 20 / 1e6:.1f} MB fp32+int64 per batch")
    t0 = time.perf_counter()
    for im, lb, y0, x0, f in samples:
        od.sample_tail(im, lb.astype(np.int32), crop, y0, x0, f, mean, std)
    t_cpu = time.perf_counter() - t0
    print(f"[tail] reference CPU tail (oracle restatement, 1 worker): {t_cpu * 1e3:.1f} ms/batch ({B / t_cpu:.0f} img/s per worker)")

    if only == "tail":
        return
    # ---------------------------------------------------------------- test-time augmentation
    nc = 19
    torch.manual_seed(0)
    m = seg_b200.DeepLab(nc, backbone="resnet101", pretrained=False, output_stride=16).cuda().eval()
    img = torch.randn(1, 3, 513, 513)
    scales = [0.75, 1.0, 1.25, 1.5, 1.75, 2.0]
    imgd = img.cuda()
    for flip in (False, True):
        ms_dev = ev_time(lambda: di.multi_scale_predict(m, imgd, scales, nc, flip=flip), 3, warm=2)
        t0 = time.perf_counter()
        with torch.no_grad():
            for _ in range(2):
                oi.multi_scale_predict(lambda t: m(t.cuda()), img, scales, nc, torch.device("cuda"), flip=flip)
        torch.cuda.synchronize()
        ms_ref = (time.perf_counter() - t0) / 2 * 1e3
        print(f"[tta] multi-scale x{len(scales)} flip={flip} 513x513/19cls DeepLab-R101: device pipeline {ms_dev:.1f} ms/image, "
              f"reference algorithm (host zoom / CPU upsample / numpy) around the same engine model {ms_ref:.1f} ms/image")
    big = torch.randn(1, 3, 1024, 2048).cuda()
    ms_dev = ev_time(lambda: di.sliding_predict(m, big, nc, flip=True), 2, warm=1)
    t0 = time.perf_counter()
    with torch.no_grad():
        oi.sliding_predict(lambda t: m(t.cuda()), big.cpu(), nc, flip=True)
    ms_ref = (time.perf_counter() - t0) * 1e3
    print(f"[tta] sliding window flip=True 1024x2048/19cls: device pipeline {ms_dev:.1f} ms/image, reference algorithm around the same "
          f"engine model {ms_ref:.1f} ms/image")

    # ---------------------------------------------------------------- optimiser
    params = [p for p in m.parameters()]
    for p in params:
        p.grad = torch.randn_like(p)
    groups = lambda: [{"params": list(m.get_decoder_params())}, {"params": list(m.get_backbone_params()), "lr": 0.001}]  # noqa: E731
    for name, cls in (("torch.optim.SGD", torch.optim.SGD), ("seg_b200.optim.SGD", FusedSGD)):
        opt = cls(groups(), lr=0.01, momentum=0.9, weight_decay=1e-4)
        ms = ev_time(opt.step, 20)
        t0 = time.perf_counter()
        for _ in range(20):
            opt.step()
        host_ms = (time.perf_counter() - t0) / 20 * 1e3
        torch.cuda.synchronize()
        n = sum(p.numel() for p in params)
        print(f"[optim] {name}.step over {len(params)} tensors / {n / 1e6:.1f} M parameters: {ms:.3f} ms on the device "
              f"({n * 20 / (ms * 1e-3) / 1e9:.0f} GB/s of the 20 B/parameter minimum), {host_ms:.3f} ms of host time to issue")


if __name__ == "__main__":
    main()
