#!/usr/bin/env python
"""Golden vectors for the validation tail and the Gaussian blur of the training tail, produced by the REFERENCE's own
BaseDataSet.__getitem__ (base/base_dataset.py) on synthetic samples:
  * val=True (`_val_augmentation`: short side -> crop_size with cv2.resize / PIL NEAREST, centre crop) on odd-sized
    portrait, landscape and square frames, down- and up-scaled, int32 labels holding -1 and 255;
  * the training chain with scale, rotate, flip and blur on, under a fixed `random` seed per sample; the draws (long side,
    angle, crop origin, flip, sigma) are recovered by replaying Python's `random` from the same seed.
Writes tests/golden/data_val_blur.npz.  Run:  SEG_REFERENCE_ROOT=<reference checkout> python tools/make_golden_val_blur.py"""
import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN, STD = [0.28689529, 0.32513294, 0.28389176], [0.17613647, 0.18099176, 0.17772235]  # dataloaders/cityscapes.py
VAL_CROP, CROP, BASE = 33, 40, 56
VAL_SIZES = [(45, 70), (71, 38), (50, 50), (21, 31), (97, 64), (33, 34), (120, 41), (29, 29)]
TRAIN_SIZES = [(45, 70), (71, 38), (50, 50), (33, 91), (64, 47), (39, 39), (80, 55), (52, 61), (47, 100), (90, 44)]


def main():
    ref = os.environ["SEG_REFERENCE_ROOT"]
    sys.path.insert(0, ref)
    for name in ("skimage", "skimage.filters"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.gaussian = lambda *a, **k: None
            sys.modules[name] = m
    from base.base_dataset import BaseDataSet

    rs = np.random.RandomState(9600)

    def sample(h, w):
        lbl = rs.randint(0, 19, (h, w)).astype(np.int32)
        lbl[rs.rand(h, w) < 0.1] = -1   # ADE20K's "no class" after its -1 shift
        lbl[rs.rand(h, w) < 0.1] = 255  # Cityscapes / VOC ignore index
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8), lbl

    val = [sample(h, w) for h, w in VAL_SIZES]
    train = [sample(h, w) for h, w in TRAIN_SIZES]
    current = []

    class Synth(BaseDataSet):
        def _set_files(self):
            self.files = list(range(16))

        def _load_data(self, index):
            im, lb = current[index]
            return im.astype(np.float32), lb, str(index)  # loaders hand float32 images on (dataloaders/cityscapes.py)

    rec = {"mean": np.asarray(MEAN), "std": np.asarray(STD), "val_crop": np.asarray(VAL_CROP), "crop": np.asarray(CROP),
           "base_size": np.asarray(BASE), "n_val": np.asarray(len(val)), "n_train": np.asarray(len(train))}
    current[:] = val
    ds = Synth(root=None, split="val", mean=MEAN, std=STD, augment=False, val=True, crop_size=VAL_CROP)
    for i, (im, lb) in enumerate(val):
        x, y = ds[i]
        rec[f"v{i}/image"], rec[f"v{i}/label"] = im, lb
        rec[f"v{i}/x"], rec[f"v{i}/y"] = x.numpy(), y.numpy()
        print("val", i, im.shape, tuple(x.shape), float(x.mean()))
    current[:] = train
    ds = Synth(root=None, split="train", mean=MEAN, std=STD, base_size=BASE, augment=True, val=False, crop_size=CROP,
               scale=True, flip=True, rotate=True, blur=True)
    for i, (im, lb) in enumerate(train):
        random.seed(500 + i)
        x, y = ds[i]
        random.seed(500 + i)  # replay: long side, angle, crop row, crop column, flip, sigma
        h0, w0 = im.shape[:2]
        longside = random.randint(int(BASE * 0.5), int(BASE * 2.0))
        h, w = (longside, int(1.0 * longside * w0 / h0 + 0.5)) if h0 > w0 else (int(1.0 * longside * h0 / w0 + 0.5), longside)
        angle = random.randint(-10, 10)
        y0 = random.randint(0, max(h, CROP) - CROP)
        x0 = random.randint(0, max(w, CROP) - CROP)
        flip = random.random() > 0.5
        sigma = random.random()
        rec[f"t{i}/image"], rec[f"t{i}/label"] = im, lb
        rec[f"t{i}/draw"] = np.asarray([h, w, angle, y0, x0, int(flip)])
        rec[f"t{i}/sigma"] = np.asarray(sigma)
        rec[f"t{i}/x"], rec[f"t{i}/y"] = x.numpy(), y.numpy()
        print("blur", i, im.shape, (h, w), angle, (y0, x0, flip), f"sigma={sigma:.3f}", float(x.mean()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "data_val_blur.npz"), **rec)


if __name__ == "__main__":
    main()
