"""oracle/data.py (CPU restatement of base_dataset.py:93-123,129-136) against golden vectors produced by the reference's
own BaseDataSet.__getitem__ (oracle/make_golden_data.py), plus the host-side draw order of seg_b200.data."""
import os
import random

import numpy as np
import torch

from oracle import data as od
from data_check import fused_emulation

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data_tail.npz")


def test_oracle_tail_is_bit_exact_against_reference():
    g = np.load(GOLD)
    crop = int(g["crop"])
    for i in range(int(g["n"])):
        y0, x0, flip = (int(v) for v in g[f"{i}/draw"])
        x, y = od.sample_tail(g[f"{i}/image"], g[f"{i}/label"], crop, y0, x0, bool(flip), g["mean"].tolist(), g["std"].tolist())
        assert torch.equal(x, torch.from_numpy(g[f"{i}/x"])), i
        assert torch.equal(y, torch.from_numpy(g[f"{i}/y"])), i


def test_draw_order_matches_reference():
    from seg_b200.data import draw_crop_flip
    g = np.load(GOLD)
    crop = int(g["crop"])
    for i in range(int(g["n"])):
        h, w = g[f"{i}/image"].shape[:2]
        random.seed(100 + i)  # the seed the golden generator gave the reference's __getitem__
        y0, x0, flip = draw_crop_flip(h, w, crop, flip=True)
        assert [y0, x0, int(flip)] == [int(v) for v in g[f"{i}/draw"]], i


def test_oracle_scaled_tail_against_reference():
    """With the random-scale resize in front (golden = the reference's BaseDataSet.__getitem__ as run, i.e. cv2.resize through
    the wheel's Intel IPP float kernels): labels (INTER_NEAREST) are exact; images agree except a small fraction of pixels
    by ONE uint8 level — IPP's closed-source float arithmetic differs from OpenCV's own code by <= 3e-3 before truncation."""
    g = np.load(GOLD)
    crop = int(g["crop"])
    mean, std = g["mean"].tolist(), g["std"].tolist()
    one_level = 1.0 / 255.0 / min(std) * 1.001
    for i in range(int(g["n"])):
        h, w, y0, x0, flip = (int(v) for v in g[f"s{i}/draw"])
        x, y = od.sample_scale_tail(g[f"{i}/image"], g[f"{i}/label"], h, w, crop, y0, x0, bool(flip), mean, std)
        assert torch.equal(y, torch.from_numpy(g[f"s{i}/y"])), i
        d = (x - torch.from_numpy(g[f"s{i}/x"])).abs()
        assert d.max().item() <= one_level, (i, d.max().item())
        assert (d > 0).float().mean().item() < 0.01, (i, (d > 0).float().mean().item())


def test_oracle_resize_is_opencvs_own_arithmetic():
    """oracle.data.cv_resize_linear_f32 / cv_resize_nearest against cv2 itself with IPP switched off: bit-exact."""
    cv2 = __import__("pytest").importorskip("cv2")
    had = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        rs = np.random.RandomState(3)
        for _ in range(40):
            sh, sw, dh, dw = int(rs.randint(5, 160)), int(rs.randint(5, 160)), int(rs.randint(3, 240)), int(rs.randint(3, 240))
            img = rs.randint(0, 256, (sh, sw, 3)).astype(np.uint8)
            lbl = rs.randint(0, 21, (sh, sw)).astype(np.int32)
            assert np.array_equal(cv2.resize(img.astype(np.float32), (dw, dh), interpolation=cv2.INTER_LINEAR), od.cv_resize_linear_f32(img, dw, dh))
            assert np.array_equal(cv2.resize(lbl, (dw, dh), interpolation=cv2.INTER_NEAREST), od.cv_resize_nearest(lbl, dw, dh))
        # the geometry of the GPU sweep: 1-pixel sources, x300 up-scales, 2000 -> 30 down-scales
        for (sh, sw, dh, dw) in ((1, 1, 7, 5), (1, 50, 13, 3), (50, 1, 2, 40), (1, 1, 300, 300), (2, 3, 600, 900),
                                 (2000, 2000, 30, 30), (2000, 37, 30, 300), (9, 2000, 1, 30)):
            img = rs.randint(0, 256, (sh, sw, 3)).astype(np.uint8)
            lbl = rs.randint(0, 21, (sh, sw)).astype(np.int32)
            assert np.array_equal(cv2.resize(img.astype(np.float32), (dw, dh), interpolation=cv2.INTER_LINEAR),
                                  od.cv_resize_linear_f32(img, dw, dh)), (sh, sw, dh, dw)
            assert np.array_equal(cv2.resize(lbl, (dw, dh), interpolation=cv2.INTER_NEAREST), od.cv_resize_nearest(lbl, dw, dh))
    finally:
        cv2.ipp.setUseIPP(had)


def test_draw_scale_matches_reference():
    from seg_b200.data import draw_crop_flip, draw_scale
    g = np.load(GOLD)
    crop, base = int(g["crop"]), int(g["base_size"])
    for i in range(int(g["n"])):
        h0, w0 = g[f"{i}/image"].shape[:2]
        random.seed(200 + i)
        h, w = draw_scale(h0, w0, base, scale=True)
        y0, x0, flip = draw_crop_flip(h, w, crop, flip=True)
        assert [h, w, y0, x0, int(flip)] == [int(v) for v in g[f"s{i}/draw"]], i


def test_oracle_rotation_is_opencvs_arithmetic():
    """oracle.data.cv_rotation_matrix / cv_warp_affine against cv2.getRotationMatrix2D / cv2.warpAffine: bit-exact, with
    IPP on or off (warpAffine's fixed-point coordinate walk is OpenCV's own code either way)."""
    cv2 = __import__("pytest").importorskip("cv2")
    rs = np.random.RandomState(8)
    extra = (45, -45, 90, -90, 180, -170)   # the GPU sweep's angles beyond the reference's draw of [-10, 10]
    for k in range(40 + 2 * len(extra)):
        h, w = int(rs.randint(20, 140)), int(rs.randint(20, 140))
        if k >= 40 and k % 2:
            h, w = (1, 1) if k % 4 == 1 else (1, 50)
        img = (rs.rand(h, w, 3) * 255).astype(np.float32)
        lbl = rs.randint(0, 21, (h, w)).astype(np.int32)
        angle = int(rs.randint(-10, 11)) if k < 40 else extra[(k - 40) // 2]
        M = od.cv_rotation_matrix((w / 2, h / 2), angle)
        assert np.array_equal(M, cv2.getRotationMatrix2D((w / 2, h / 2), angle, 1.0))
        assert np.array_equal(cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR), od.cv_warp_affine(img, M, w, h, True))
        assert np.array_equal(cv2.warpAffine(lbl, M, (w, h), flags=cv2.INTER_NEAREST), od.cv_warp_affine(lbl, M, w, h, False))


def test_oracle_scale_rotate_tail_against_reference():
    """The whole default augmentation chain of config.json minus blur — scale, rotate, pad, crop, flip, ToTensor, Normalize —
    against the reference's BaseDataSet.__getitem__ as run: labels exact, images within one uint8 level on < 1 % of the
    pixels (the IPP float resize, see above; the rotation itself is restated exactly)."""
    g = np.load(GOLD)
    crop = int(g["crop"])
    mean, std = g["mean"].tolist(), g["std"].tolist()
    one_level = 1.0 / 255.0 / min(std) * 1.001
    for i in range(int(g["n"])):
        h, w, angle, y0, x0, flip = (int(v) for v in g[f"r{i}/draw"])
        x, y = od.sample_scale_tail(g[f"{i}/image"], g[f"{i}/label"], h, w, crop, y0, x0, bool(flip), mean, std, angle=angle)
        assert torch.equal(y, torch.from_numpy(g[f"r{i}/y"])), i
        d = (x - torch.from_numpy(g[f"r{i}/x"])).abs()
        assert d.max().item() <= one_level, (i, d.max().item())
        assert (d > 0).float().mean().item() < 0.01, (i, (d > 0).float().mean().item())


def test_fused_scale_rotate_formulation_equals_staged_oracle():
    """The experimental kernel computes every output pixel from the raw sample in one go (no resized / rotated image).  Its
    numpy transcription must equal the staged oracle (resize, then warpAffine, then the tail) bit for bit — with and without
    a rotation — which pins the fusion logic the CUDA code follows line by line."""
    g = np.load(GOLD)
    crop = int(g["crop"])
    mean, std = g["mean"].tolist(), g["std"].tolist()
    for i in range(int(g["n"])):
        h, w, angle, y0, x0, flip = (int(v) for v in g[f"r{i}/draw"])
        for ang in (angle, None, -10, 0):
            x, y = fused_emulation(g[f"{i}/image"], g[f"{i}/label"], h, w, ang, crop, y0, x0, bool(flip), mean, std)
            rx, ry = od.sample_scale_tail(g[f"{i}/image"], g[f"{i}/label"], h, w, crop, y0, x0, bool(flip), mean, std, angle=ang)
            assert torch.equal(y, ry), (i, ang)
            assert torch.equal(x, rx), (i, ang, (x - rx).abs().max().item())


def test_draw_order_with_rotation_matches_reference():
    from seg_b200.data import draw_crop_flip, draw_rotate, draw_scale
    g = np.load(GOLD)
    crop, base = int(g["crop"]), int(g["base_size"])
    for i in range(int(g["n"])):
        h0, w0 = g[f"{i}/image"].shape[:2]
        random.seed(300 + i)  # the seed the golden generator gave the reference's __getitem__ (scale + rotate on)
        h, w = draw_scale(h0, w0, base, scale=True)
        angle = draw_rotate(True)
        y0, x0, flip = draw_crop_flip(h, w, crop, flip=True)
        assert [h, w, angle, y0, x0, int(flip)] == [int(v) for v in g[f"r{i}/draw"]], i
