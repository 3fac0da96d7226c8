"""Label maps in the augmentation kernels and the device loaders on the H100.

* Mapped arenas (SEG_AUG_LABEL_MAP records: uint8 label + 256-entry id table) from every kernel — plain tail, scale, full,
  full + blur, val — are bit-identical to the staged CPU oracle run on the host-mapped labels, padded crops included,
  whose fill is the post-map 0 and not map[0].
* Unflagged records give the same bytes under the mapped twins as under the existing entry points (whose SASS is
  unchanged, DESIGN.md §7), and those match the oracle bit for bit.
* The overlay DataPrefetcher against the reference's, and `python -m seg_b200.launch train.py` end to end, on seeded
  synthetic trees (reference from oracle/_ref/reference.zip; skipped where build() had none to pack)."""
import json
import math
import os
import re
import subprocess
import sys
import zipfile

import numpy as np
import pytest
import torch

from oracle import data as od
import val_blur_oracle as vbo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
needs_ref = pytest.mark.skipif(not os.path.isfile(REF_ZIP), reason="oracle/_ref/reference.zip not built (build() found no reference checkout)")
MEAN, STD = [0.28689529, 0.32513294, 0.28389176], [0.17613647, 0.18099176, 0.17772235]
CROP = 40


def bits(t):
    return t.contiguous().view(torch.int32)


def id_table(seed):
    """A Cityscapes-like table: map[0] = 255 (so a fill read through the map would show), negative and large entries."""
    t = np.random.default_rng(seed).integers(-1, 300, 256).astype(np.int32)
    t[0] = 255
    return t


def raw_samples(seed, sizes=((24, 30), (52, 64), (40, 33), (70, 90))):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        lb = rng.integers(0, 256, (h, w), dtype=np.uint8)
        lb[0, :] = 0   # id 0 inside the image maps to 255; the padding must stay 0
        out.append((im, lb))
    return out


def batcher():
    from seg_b200.data import DeviceBatcher
    return DeviceBatcher(MEAN, STD, CROP, "cuda:0", max_bytes=8 << 20)


def compare(case, got, want):
    x, y = got
    torch.cuda.synchronize()
    for b, (wx, wy) in enumerate(want):
        assert torch.equal(bits(x[b].cpu()), bits(wx)), f"{case}: sample {b}: image differs from the oracle"
        assert torch.equal(y[b].cpu(), wy), f"{case}: sample {b}: label differs from the oracle"


def cases(seed, table):
    """(kind, samples for the batcher, per-sample oracle) for every kernel, with the label read through `table`."""
    rng = np.random.default_rng(seed)
    raw = raw_samples(seed)
    mapped = [(im, table[lb] if table is not None else lb) for im, lb in raw]
    plain, scale, full, sig = [], [], [], []
    for k, (im, lb) in enumerate(raw):
        H, W = im.shape[:2]
        h, w = (int(H * 0.8) + 1, int(W * 0.8) + 1) if k % 2 else (int(H * 1.3), int(W * 1.3))
        ph, pw = max(H, CROP), max(W, CROP)
        y0, x0 = int(rng.integers(0, ph - CROP + 1)), int(rng.integers(0, pw - CROP + 1))
        plain.append((im, lb, y0, x0, bool(k % 2)))
        y1, x1 = int(rng.integers(0, max(h, CROP) - CROP + 1)), int(rng.integers(0, max(w, CROP) - CROP + 1))
        scale.append((im, lb, h, w, y1, x1, bool(k % 2)))
        full.append((im, lb, h, w, [-10, 7, 0, 3][k], y1, x1, bool(k % 2)))
        sig.append([0.9, None, 0.5, 0.2][k])
    want_plain = [od.sample_tail(mim, mlb, CROP, y0, x0, f, MEAN, STD) for (mim, mlb), (_, _, y0, x0, f) in zip(mapped, plain)]
    want_scale = [vbo.sample_blur_tail(mim, mlb, h, w, CROP, y0, x0, f, MEAN, STD)
                  for (mim, mlb), (_, _, h, w, y0, x0, f) in zip(mapped, scale)]
    want_full = [vbo.sample_blur_tail(mim, mlb, h, w, CROP, y0, x0, f, MEAN, STD, angle=a)
                 for (mim, mlb), (_, _, h, w, a, y0, x0, f) in zip(mapped, full)]
    want_blur = [vbo.sample_blur_tail(mim, mlb, h, w, CROP, y0, x0, f, MEAN, STD, angle=a, sigma=s)
                 for (mim, mlb), (_, _, h, w, a, y0, x0, f), s in zip(mapped, full, sig)]
    want_val = [vbo.sample_val_tail(mim, np.asarray(mlb, np.int32), CROP, MEAN, STD) for mim, mlb in mapped]
    return [("plain", plain, None, want_plain), ("scale", scale, None, want_scale), ("full", full, None, want_full),
            ("full_blur", full, sig, want_blur), ("val", raw, None, want_val)]


def stage(b, kind, samples, sigmas, table):
    if kind == "plain":
        return b.stage(samples, label_map=table)
    if kind == "scale":
        return b.stage_scaled(samples, label_map=table)
    if kind in ("full", "full_blur"):
        return b.stage_full(samples, sigmas, label_map=table)
    return b.stage_val(samples, label_map=table)


@pytest.mark.parametrize("seed", [1, 2])
def test_mapped_arenas_match_the_staged_oracle(seed):
    b = batcher()
    t = id_table(seed)
    for kind, samples, sigmas, want in cases(seed, t):
        got = stage(b, kind, samples, sigmas, t)
        compare(f"mapped {kind}", got, want)   # sample 0 (24 x 30) is padded: the oracle pads the MAPPED label with 0


def test_padded_cityscapes_crop_fills_with_class_0():
    """A 20 x 24 Cityscapes sample of id 0 only (map[0] = 255, ignore) in a 40 x 40 crop: 255 inside, 0 in the padding —
    the reference remaps in _load_data, before copyMakeBorder(value=0)."""
    t = id_table(0)
    im = np.full((20, 24, 3), 100, np.uint8)
    lb = np.zeros((20, 24), np.uint8)
    b = batcher()
    for kind in ("plain", "scale", "full"):
        if kind == "plain":
            _, y = b.stage([(im, lb, 0, 0, False)], label_map=t)
        elif kind == "scale":
            _, y = b.stage_scaled([(im, lb, 20, 24, 0, 0, False)], label_map=t)
        else:
            _, y = b.stage_full([(im, lb, 20, 24, 5, 0, 0, False)], label_map=t)
        y = y[0].cpu()
        assert (y[20:, :] == 0).all() and (y[:, 24:] == 0).all(), kind
        assert (y[2:18, 2:22] == 255).all(), kind


@pytest.mark.parametrize("seed", [3])
def test_unflagged_records_are_unchanged(seed):
    """Records without the flag: the existing entry points match the oracle bit for bit, and the mapped twins give the
    same bytes for them."""
    from seg_b200 import data
    b = batcher()
    for kind, samples, sigmas, want in cases(seed, None):
        got = stage(b, kind, samples, sigmas, None)
        compare(f"unflagged {kind}", got, want)
        pack = {"plain": lambda: data.pack_plain(samples, CROP), "scale": lambda: data.pack_scaled(samples, CROP),
                "full": lambda: data.pack_full(samples, CROP), "full_blur": lambda: data.pack_full(samples, CROP, sigmas),
                "val": lambda: data.pack_val(samples, CROP)}[kind]()
        assert pack.kind == kind and not pack.label_map
        dev = pack.arena.cuda()
        pack.label_map = True   # the mapped instantiation on records without the flag
        twin = data.launch_packed(pack, dev, MEAN, STD)
        torch.cuda.synchronize()
        assert torch.equal(bits(twin[0]), bits(got[0])) and torch.equal(twin[1], got[1]), f"{kind}: mapped twin differs"


def extract_reference(tmp_path):
    ref = tmp_path / "reference"
    with zipfile.ZipFile(REF_ZIP) as z:
        z.extractall(ref)
    return ref


@needs_ref
def test_overlay_prefetcher_matches_the_reference_prefetcher(tmp_path):
    ref = extract_reference(tmp_path)
    data = tmp_path / "data"
    data.mkdir()
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "pytorch-segmentation_b200"))
    env.pop("SEG_DEVICE_DATA", None)
    r = subprocess.run([sys.executable, "-W", "ignore", os.path.join(ROOT, "tests", "device_loader_check.py"), str(ref), str(data), "gpu"],
                       env=env, cwd=str(ref), capture_output=True, text=True, timeout=1800)
    print(r.stdout[-3000:])
    assert "CHECK_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]


@needs_ref
def test_train_py_end_to_end_on_the_device_loaders(tmp_path):
    """The unmodified train.py through seg_b200.launch on a synthetic Cityscapes tree: one epoch with validation, the
    loaders and DataPrefetcher from the overlay; finite validation loss and mIoU are logged."""
    import device_loader_check as dlc
    ref = extract_reference(tmp_path)
    tree = dlc.make_cityscapes(str(tmp_path / "cityscapes"), n=8)
    cfg = json.load(open(ref / "config.json"))
    cfg["arch"]["args"].update(backbone="resnet50", pretrained=False)
    for k in ("train_loader", "val_loader"):
        cfg[k]["args"].update(data_dir=tree, batch_size=4, num_workers=2)
    cfg["train_loader"]["args"].update(base_size=80, crop_size=64)
    cfg["val_loader"]["args"].update(crop_size=64)
    cfg["trainer"].update(epochs=1, val_per_epochs=1, save_dir=str(tmp_path / "saved"), log_dir=str(tmp_path / "runs"), save_period=1)
    p = tmp_path / "config.json"
    p.write_text(json.dumps(cfg))
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "pytorch-segmentation_b200"))
    env.pop("SEG_DEVICE_DATA", None)
    r = subprocess.run([sys.executable, "-W", "ignore", "-m", "seg_b200.launch", "train.py", "-c", str(p)], env=env, cwd=str(ref),
                       capture_output=True, text=True, timeout=1800)
    out = r.stdout + r.stderr
    print(out[-3000:])
    assert r.returncode == 0, out[-5000:]
    loss = re.findall(r"val_loss\s*:\s*([-+0-9.eEna]+)", out)
    miou = re.findall(r"Mean_IoU\s*:\s*([-+0-9.eEna]+)", out)
    assert loss and miou, out[-3000:]
    assert math.isfinite(float(loss[-1])) and math.isfinite(float(miou[-1])), (loss, miou)
