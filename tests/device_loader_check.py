"""Shared by the device-loader tests: seeded synthetic Cityscapes / VOC / ADE20K trees, the CPU oracle of one
DeviceSample (the draws a device-mode dataset returned, staged through oracle/data.py and the blur / val oracle), and the
reference-vs-overlay comparisons.  Run as a script in a fresh interpreter (the reference's `base` / `utils` / `models`
packages must be resolved through the overlay):  python device_loader_check.py <reference root> <data dir> <check> [device]"""
import os
import random
import sys

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

CROP = 48
SIZES = [(40, 56), (64, 96), (72, 50), (33, 47), (96, 120), (50, 40)]   # several smaller than the crop: padding appears


def _rgb(rng, h, w):
    base = rng.integers(0, 256, (h // 4 + 1, w // 4 + 1, 3)).astype(np.uint8)   # smooth-ish so interpolation matters
    img = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR))
    return np.clip(img.astype(np.int32) + rng.integers(-6, 7, img.shape), 0, 255).astype(np.uint8)


def make_cityscapes(root, seed=0, n=6):
    rng = np.random.default_rng(seed)
    for split in ("train", "val"):
        di = os.path.join(root, "leftImg8bit_trainvaltest", "leftImg8bit", split, "city0")
        dl = os.path.join(root, "gtFine_trainvaltest", "gtFine", split, "city0")
        os.makedirs(di, exist_ok=True)
        os.makedirs(dl, exist_ok=True)
        for k in range(n):
            h, w = SIZES[k % len(SIZES)]
            Image.fromarray(_rgb(rng, h, w)).save(os.path.join(di, f"city0_{k:06d}_000019_leftImg8bit.png"))
            lab = rng.integers(0, 256, (h, w)).astype(np.uint8)   # every id, the unlabelled ones included
            lab[: h // 3] = rng.integers(0, 34, (h // 3, w))
            Image.fromarray(lab, mode="L").save(os.path.join(dl, f"city0_{k:06d}_000019_gtFine_labelIds.png"))
    return root


def make_voc(root, seed=1, n=6):
    rng = np.random.default_rng(seed)
    base = os.path.join(root, "VOCdevkit", "VOC2012")
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
        os.makedirs(os.path.join(base, d), exist_ok=True)
    ids = [f"2007_{k:06d}" for k in range(n)]
    for k, i in enumerate(ids):
        h, w = SIZES[k % len(SIZES)]
        Image.fromarray(_rgb(rng, h, w)).save(os.path.join(base, "JPEGImages", i + ".jpg"), quality=95)
        lab = rng.integers(0, 21, (h, w)).astype(np.uint8)
        lab[:, : w // 5] = 255
        p = Image.fromarray(lab, mode="P")
        p.putpalette(list(range(256)) * 3)
        p.save(os.path.join(base, "SegmentationClass", i + ".png"))
    for split in ("train", "val"):
        with open(os.path.join(base, "ImageSets/Segmentation", split + ".txt"), "w") as f:
            f.write("\n".join(ids) + "\n")
    return root


def make_ade20k(root, seed=2, n=6):
    rng = np.random.default_rng(seed)
    for split in ("training", "validation"):
        di, dl = os.path.join(root, "images", split), os.path.join(root, "annotations", split)
        os.makedirs(di, exist_ok=True)
        os.makedirs(dl, exist_ok=True)
        for k in range(n):
            h, w = SIZES[k % len(SIZES)]
            Image.fromarray(_rgb(rng, h, w)).save(os.path.join(di, f"ADE_{k:08d}.jpg"), quality=95)
            Image.fromarray(rng.integers(0, 151, (h, w)).astype(np.uint8), mode="L").save(os.path.join(dl, f"ADE_{k:08d}.png"))
    return root


def oracle_sample(s, mean, std):
    """The CPU oracle of one DeviceSample: the label map applied on the host first (where _load_data applies it), then the
    reference's staged augmentation.  Returns (fp32 [3,c,c], int64 [c,c])."""
    import val_blur_oracle as vbo
    from oracle import data as od
    image, label, draws, crop, lmap = s
    lab = lmap[label] if lmap is not None else np.asarray(label, dtype=np.int32)
    if draws is None:
        return vbo.sample_val_tail(image, lab.astype(np.int32), crop, mean, std)
    h, w, angle, y0, x0, flip, sigma = draws
    H, W = image.shape[:2]
    if h is None and angle is None and sigma is None:
        return od.sample_tail(image, lab, crop, y0, x0, flip, mean, std)
    return vbo.sample_blur_tail(image, lab, h if h is not None else H, w if w is not None else W, crop, y0, x0, flip, mean, std,
                                angle=angle, sigma=sigma)


def within_one_level(x, ref, std):
    """Images identical or off by one uint8 level (1/255/std after Normalize); returns the share of values off."""
    import torch
    d = (x - ref).abs()
    lvl = torch.as_tensor([1.0 / 255 / v for v in std], dtype=torch.float32).view(-1, 1, 1)
    lvl = lvl.expand_as(d) if d.dim() == 3 else lvl.unsqueeze(0).expand_as(d)
    off = d > 1e-6
    assert bool((d[off] <= lvl[off] * 1.001 + 1e-6).all()), f"image differs by more than one level: max {float(d.max())}"
    return float(off.float().mean())


CONFIGS = {   # loader kwargs on top of data_dir / batch_size / split / crop_size
    "plain": dict(augment=True, flip=True, scale=False),
    "scale": dict(augment=True, base_size=80, scale=True, flip=True),
    "rotate": dict(augment=True, base_size=80, scale=True, flip=True, rotate=True),
    "rotate_noscale": dict(augment=True, flip=True, rotate=True),
    "blur": dict(augment=True, base_size=80, scale=True, flip=True, rotate=True, blur=True),
    "blur_only": dict(augment=True, flip=False, blur=True),
    "val": dict(val=True),
}
DATASETS = {"CityScapes": ("train", "val"), "VOC": ("train", "val"), "ADE20K": ("training", "validation")}
EXPECTED_KIND = {"plain": {"plain"}, "scale": {"scale"}, "rotate": {"full"}, "rotate_noscale": {"full"},
                 "blur": {"full", "full_blur"}, "blur_only": {"plain", "full_blur"}, "val": {"val"}}


def _reference_modules(ref_root):
    """The reference's own dataloaders package, loaded privately next to the overlay's."""
    import importlib.util
    import types
    pkg = types.ModuleType("_refdl")
    pkg.__path__ = [os.path.join(ref_root, "dataloaders")]
    sys.modules["_refdl"] = pkg
    out = {}
    for name, mod in (("CityScapes", "cityscapes"), ("VOC", "voc"), ("ADE20K", "ade20k")):
        spec = importlib.util.spec_from_file_location(f"_refdl.{mod}", os.path.join(ref_root, "dataloaders", mod + ".py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        out[name] = getattr(m, name)
    return out


def loaders(ref_root, data_dirs, name, config, workers, batch=3):
    import dataloaders
    ref = _reference_modules(ref_root)[name]
    train, val = DATASETS[name]
    kw = dict(data_dir=data_dirs[name], batch_size=batch, split=val if config == "val" else train, crop_size=CROP,
              num_workers=workers, shuffle=True, **CONFIGS[config])
    return ref(**kw), getattr(dataloaders, name)(**kw)


def check_datasets(ref_root, data_dirs, exact=False):
    """num_workers=0 and 2: every overlay sample, staged through the oracle, against the reference's sample.  Labels are
    identical; images within one level on under 1 % of the values as OpenCV runs by default, identical with OpenCV's
    IPP and SIMD dispatch off (exact=True)."""
    import torch
    from seg_b200.data import DeviceSample, PackedBatch, device_collate
    stats = []
    for name in DATASETS:
        for config in CONFIGS:
            for workers in (0, 2):
                r, o = loaders(ref_root, data_dirs, name, config, workers)
                assert o.dataset.device_mode and not hasattr(r.dataset, "device_mode")
                assert len(o) == len(r) and o.MEAN == r.MEAN and o.batch_size == r.batch_size
                assert o.dataset.num_classes == r.dataset.num_classes and o.dataset.palette == r.dataset.palette
                o.collate_fn = _tee   # the workers return the samples next to the packed batch
                torch.manual_seed(7)   # the shuffle and, in workers, each worker's `random` seed
                random.seed(7)         # num_workers=0: the draws come from this process's `random`
                rb = list(r)
                torch.manual_seed(7)
                random.seed(7)
                ob = list(o)
                assert len(rb) == len(ob)
                for (x, y), (pb, samples) in zip(rb, ob):
                    assert isinstance(pb, PackedBatch) and all(isinstance(s, DeviceSample) for s in samples)
                    assert pb.kind in EXPECTED_KIND[config], (name, config, pb.kind)
                    again = device_collate(samples)
                    assert again.kind == pb.kind and torch.equal(again.arena, pb.arena), "packing is not deterministic"
                    for b, s in enumerate(samples):
                        ox, oy = oracle_sample(s, o.MEAN, o.STD)
                        assert torch.equal(oy, y[b]), f"{name}/{config}/w{workers}: labels differ from the reference"
                        stats.append(within_one_level(ox, x[b], o.STD))
                print(f"{name} {config} workers={workers}: {len(rb)} batches, kinds ok")
    share = float(np.mean(stats))
    print(f"image values one level off: {share:.5f} overall, {max(stats):.4f} in the worst sample")
    assert share == 0.0 if exact else share < 0.01


def _tee(batch):
    from seg_b200.data import device_collate
    return device_collate(batch), list(batch)


def check_cityscapes_table(ref_root):
    """The table equals the reference's _load_data over all 256 values (one label PNG holding every value)."""
    import tempfile
    from dataloaders._device import cityscapes_label_map
    ref = _reference_modules(ref_root)["CityScapes"]
    with tempfile.TemporaryDirectory() as d:
        make_cityscapes(d, n=1)
        lp = os.path.join(d, "gtFine_trainvaltest", "gtFine", "train", "city0", "city0_000000_000019_gtFine_labelIds.png")
        raw = np.arange(256, dtype=np.uint8).reshape(16, 16)
        Image.fromarray(raw, mode="L").save(lp)
        ip = lp.replace("gtFine_trainvaltest", "leftImg8bit_trainvaltest").replace("gtFine", "leftImg8bit", 1)
        ip = ip.replace("_gtFine_labelIds", "_leftImg8bit")
        Image.fromarray(np.zeros((16, 16, 3), np.uint8)).save(ip)
        ds = ref(data_dir=d, batch_size=1, split="train").dataset
        _, lab, _ = ds._load_data(0)
    t = cityscapes_label_map()
    assert np.array_equal(t[raw], lab), "the 256-entry table differs from the reference's per-pixel loop"
    assert t[0] == 255 and t[7] == 0 and t[33] == 18
    print("cityscapes table ok")


def check_fallback(ref_root, data_dirs):
    import torch
    import dataloaders
    d = data_dirs["CityScapes"]
    cases = [dict(crop_size=None, augment=True), dict(crop_size=0, augment=True), dict(crop_size=CROP, augment=False),
             dict(crop_size=CROP, augment=True, return_id=True)]
    for kw in cases:
        o = dataloaders.CityScapes(data_dir=d, batch_size=1, split="train", **kw)
        assert not o.dataset.device_mode, kw
        item = o.dataset[0]
        assert isinstance(item[0], torch.Tensor) and item[0].is_floating_point(), kw
    os.environ["SEG_DEVICE_DATA"] = "0"
    try:
        o = dataloaders.CityScapes(data_dir=d, batch_size=1, split="train", crop_size=CROP, augment=True)
        assert not o.dataset.device_mode
    finally:
        del os.environ["SEG_DEVICE_DATA"]
    print("fallback ok")


def check_overlay_names(ref_root):
    import base
    import dataloaders
    from seg_b200.data import DevicePrefetcher
    ref_base = os.path.join(ref_root, "base")
    assert base.DataPrefetcher is DevicePrefetcher
    for n in ("BaseModel", "BaseTrainer", "BaseDataSet", "BaseDataLoader"):
        assert getattr(base, n).__module__.startswith("base."), n
        assert os.path.dirname(sys.modules[getattr(base, n).__module__].__file__) == ref_base, n
    assert dataloaders.COCO.__module__ == "dataloaders.coco" and dataloaders.DeepScene.__module__ == "dataloaders.deepscene"
    assert issubclass(dataloaders.CityScapes, base.BaseDataLoader)
    print("overlay names ok")


def check_prefetchers(ref_root, data_dirs):
    """The overlay's DataPrefetcher over the overlay loaders against the reference's DataPrefetcher over the reference's
    loaders (num_workers=2, the same seeds): device batches with identical labels, images within one level."""
    import torch
    import base
    from base.base_dataloader import DataPrefetcher as RefPrefetcher   # the reference's class (base/base_dataloader.py)
    assert RefPrefetcher is not base.DataPrefetcher
    stats = []
    for name in DATASETS:
        for config in CONFIGS:
            r, o = loaders(ref_root, data_dirs, name, config, 2)
            torch.manual_seed(11)
            rb = [(x.clone(), y.clone()) for x, y in RefPrefetcher(r, device=torch.device("cuda:0"))]
            torch.manual_seed(11)
            ob = [(x.clone(), y.clone()) for x, y in base.DataPrefetcher(o, device=torch.device("cuda:0"))]
            assert len(rb) == len(ob) == len(o)
            for (x, y), (ox, oy) in zip(rb, ob):
                assert ox.is_cuda and ox.dtype == torch.float32 and oy.dtype == torch.int64 and ox.shape == x.shape
                assert torch.equal(oy, y), f"{name}/{config}: device labels differ from the reference's"
                stats.append(within_one_level(ox.cpu(), x.cpu(), o.STD))
            print(f"prefetcher {name} {config}: {len(rb)} batches")
    share = float(np.mean(stats))
    print(f"prefetcher image values one level off: {share:.5f} overall")
    assert share < 0.01


def build_trees(d):
    return {"CityScapes": make_cityscapes(os.path.join(d, "cityscapes")), "VOC": make_voc(os.path.join(d, "voc")),
            "ADE20K": make_ade20k(os.path.join(d, "ade20k"))}


if __name__ == "__main__":
    ref_root, data_dir, check = sys.argv[1], sys.argv[2], sys.argv[3]
    from seg_b200 import launch
    launch.setup_paths(ref_root)
    random.seed(0)
    trees = build_trees(data_dir)
    if check == "cpu":
        check_overlay_names(ref_root)
        check_cityscapes_table(ref_root)
        check_fallback(ref_root, trees)
        check_datasets(ref_root, trees)
    elif check == "cpu_exact":
        import cv2
        cv2.setUseOptimized(False)   # OpenCV's own C++ paths, which the oracle restates (workers inherit it by fork)
        cv2.ipp.setUseIPP(False)
        check_datasets(ref_root, trees, exact=True)
    elif check == "gpu":
        check_prefetchers(ref_root, trees)
    print("CHECK_OK")
