"""The `base` and `dataloaders` overlays against the unmodified reference (oracle/_ref/reference.zip, extracted to a
temporary directory; skipped where build() had no reference checkout to pack): seeded synthetic Cityscapes, VOC and
ADE20K trees, the reference's loaders and the overlay's at num_workers 0 and 2, every overlay sample staged through the
CPU oracle.  The checks themselves are in tests/device_loader_check.py, run in a fresh interpreter because the overlay
resolves the reference's packages through sys.path."""
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")
CHECK = os.path.join(ROOT, "tests", "device_loader_check.py")
needs_ref = pytest.mark.skipif(not os.path.isfile(REF_ZIP), reason="oracle/_ref/reference.zip not built (build() found no reference checkout)")


def run_check(tmp_path, check):
    ref = tmp_path / "reference"
    with zipfile.ZipFile(REF_ZIP) as z:
        z.extractall(ref)
    data = tmp_path / "data"
    data.mkdir()
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "pytorch-segmentation_b200")
    env.pop("SEG_DEVICE_DATA", None)
    r = subprocess.run([sys.executable, "-W", "ignore", CHECK, str(ref), str(data), check], env=env, cwd=str(ref), capture_output=True,
                       text=True, timeout=1800)
    assert "CHECK_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
    return r.stdout


@needs_ref
def test_overlay_loaders_match_the_reference(tmp_path):
    """Overlay names, the Cityscapes table over all 256 values, the fallback cases, and train (scale / rotate / flip /
    blur on and off, padded crops) and val batches: labels identical, images within one level on < 1 % of the values."""
    out = run_check(tmp_path, "cpu")
    for line in ("overlay names ok", "cityscapes table ok", "fallback ok", "ADE20K val workers=2"):
        assert line in out


@needs_ref
def test_overlay_loaders_are_exact_with_opencvs_own_paths(tmp_path):
    """With OpenCV's IPP and SIMD dispatch off the reference runs the arithmetic the oracle restates: images identical."""
    assert "0.00000 overall" in run_check(tmp_path, "cpu_exact")


@needs_ref
def test_overlay_test_assertions_hold_with_the_new_packages(tmp_path):
    """tests/test_overlay_cpu.py's registry assertions, with `base` and `dataloaders` now coming from the overlay."""
    import test_overlay_cpu
    test_overlay_cpu.test_overlay_resolves_registries(tmp_path)


def test_packer_layout_and_label_map_flag():
    """pack_arena: records, images and labels 4-byte aligned, the 256-entry table after a flagged uint8 label, the PIL
    index tables after the table; lbl_bytes other than 1, 4 and 1 | AUG_LABEL_MAP, and a table with int32 labels, refused."""
    from seg_b200 import data, lib
    rng = np.random.default_rng(0)
    im = rng.integers(0, 256, (5, 7, 3), dtype=np.uint8)
    lb = rng.integers(0, 256, (5, 7), dtype=np.uint8)
    t = np.arange(256, dtype=np.int32)[::-1].copy()
    pb = data.pack_val([(im, lb), (im, lb)], 4, label_map=t)
    a = pb.arena.numpy()
    rec = np.frombuffer(a[:2 * data._SCALE_ENTRY.itemsize].tobytes(), dtype=data._SCALE_ENTRY)
    assert pb.kind == "val" and pb.label_map and (rec["lbl_bytes"] == 1 | lib.AUG_LABEL_MAP).all()
    for r in rec:
        assert r["img_off"] % 4 == 0 and r["lbl_off"] % 4 == 0
        assert np.array_equal(a[r["img_off"]:r["img_off"] + im.size], im.reshape(-1))
        assert np.array_equal(a[r["lbl_off"]:r["lbl_off"] + lb.size], lb.reshape(-1))
        m = r["lbl_off"] + (lb.size + 3) // 4 * 4
        assert np.array_equal(np.frombuffer(a[m:m + 1024].tobytes(), np.int32), t)
        h, w = int(r["h"]), int(r["w"])
        tabs = np.frombuffer(a[m + 1024:m + 1024 + 4 * (w + h)].tobytes(), np.int32)
        assert np.array_equal(tabs, np.concatenate([data.pil_nearest_index(7, w), data.pil_nearest_index(5, h)]))
    plain = data.pack_plain([(im, lb, 0, 0, False)], 4)
    assert not plain.label_map and np.frombuffer(plain.arena.numpy()[:data._ENTRY.itemsize].tobytes(), data._ENTRY)["lbl_bytes"][0] == 1
    with pytest.raises(ValueError, match="uint8 labels"):
        data.pack_plain([(im, lb.astype(np.int32), 0, 0, False)], 4, label_map=t)
    with pytest.raises(ValueError, match="256"):
        data.pack_plain([(im, lb, 0, 0, False)], 4, label_map=t[:255])
    with pytest.raises(ValueError, match="lbl_bytes"):
        data.pack_arena([(im, lb)], data._ENTRY, lambda b, io, lo, H, W, l: (io, lo, H, W, 0, 0, 0, 2))
    with pytest.raises(RuntimeError, match="max_bytes"):
        import torch
        data.pack_plain([(im, lb, 0, 0, False)], 4, out=torch.empty(64, dtype=torch.uint8))


def test_collate_picks_the_kernel_from_the_draws():
    from seg_b200 import data
    im = np.zeros((30, 40, 3), np.uint8)
    lb = np.zeros((30, 40), np.uint8)
    S = lambda d: data.DeviceSample(im, lb, d, 24, None)  # noqa: E731
    assert data.device_collate([S((None, None, None, 0, 0, False, None))] * 2).kind == "plain"
    assert data.device_collate([S((None, None, None, 0, 0, False, 0.2))] * 2).kind == "plain"    # k = 1: no blur
    assert data.device_collate([S((36, 48, None, 0, 0, True, None))] * 2).kind == "scale"
    assert data.device_collate([S((36, 48, None, 0, 0, True, None)), S((None, None, 5, 1, 2, False, None))]).kind == "full"
    assert data.device_collate([S((None, None, None, 0, 0, False, 0.2)), S((None, None, None, 0, 0, False, 0.9))]).kind == "full_blur"
    assert data.device_collate([S(None)] * 2).kind == "val"
    with pytest.raises(ValueError, match="mixes"):
        data.device_collate([S(None), S((None, None, None, 0, 0, False, None))])
