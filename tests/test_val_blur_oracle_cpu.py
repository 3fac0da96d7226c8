"""The validation tail and the Gaussian blur of the training tail: tests/val_blur_oracle.py against cv2 / PIL over random
size pairs and sigmas, and against golden vectors from the reference's own BaseDataSet.__getitem__
(tools/make_golden_val_blur.py); plus the host-side geometry and draws of seg_b200.data."""
import math
import os
import random

import numpy as np
import pytest
import torch

import val_blur_oracle as vo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data_val_blur.npz")


def test_pil_nearest_restatement_is_bit_exact_against_pillow():
    Image = pytest.importorskip("PIL.Image")
    rs = np.random.RandomState(12)
    pairs = [(int(rs.randint(1, 300)), int(rs.randint(1, 300)), int(rs.randint(1, 700)), int(rs.randint(1, 700))) for _ in range(400)]
    pairs += [(1024, 2048, 480, 960), (2048, 1024, 960, 480), (1, 1, 5, 9), (7, 1, 1, 3), (2000, 37, 30, 300), (480, 480, 480, 480)]
    closed_form_differs = 0
    for k, (H, W, h, w) in enumerate(pairs):
        lbl = rs.randint(-5, 300, (H, W)).astype(np.int32)
        got = np.asarray(Image.fromarray(lbl).resize((w, h), resample=Image.NEAREST), dtype=np.int32)
        assert Image.fromarray(lbl).mode == "I"
        assert np.array_equal(vo.pil_resize_nearest(lbl, w, h), got), (H, W, h, w)
        if k % 4 == 0:  # mode "L" follows the same rule
            l8 = (lbl & 255).astype(np.uint8)
            assert np.array_equal(vo.pil_resize_nearest(l8, w, h), np.asarray(Image.fromarray(l8).resize((w, h), Image.NEAREST)))
        cf = lambda s, d: np.minimum(np.floor((np.arange(d) + 0.5) * (s / d)).astype(int), s - 1)  # noqa: E731
        closed_form_differs += not np.array_equal(lbl[cf(H, h)][:, cf(W, w)], got)
    # why the index is replayed rather than computed in closed form
    assert closed_form_differs > len(pairs) // 4, closed_form_differs


def test_device_index_tables_equal_the_restatement():
    from seg_b200.data import pil_nearest_index
    rs = np.random.RandomState(13)
    for _ in range(200):
        H, W, h, w = (int(v) for v in rs.randint(1, 900, 4))
        lbl = np.arange(H * W, dtype=np.int32).reshape(H, W)
        assert np.array_equal(lbl[pil_nearest_index(H, h)][:, pil_nearest_index(W, w)], vo.pil_resize_nearest(lbl, w, h))


def test_gaussian_taps_are_getGaussianKernel():
    cv2 = pytest.importorskip("cv2")
    from seg_b200.data import gaussian_taps
    rs = np.random.RandomState(14)
    sigmas = list(0.6061 + rs.rand(20000) * (1.2121 - 0.6061)) + [2 / 3.3 + 1e-12, 0.61, 0.999999, 1.0, 1.2]
    for s in sigmas:
        g = cv2.getGaussianKernel(3, s, cv2.CV_32F).ravel()
        assert vo.blur_ksize(s) == 3
        k0, k1 = vo.cv_gaussian_taps(s)
        assert g[1] == k0 and g[0] == k1 and g[2] == k1, s
        assert gaussian_taps(s) == (float(k0), float(k1))
    for s in (0.0, 0.3, 0.6, 2 / 3.3 - 1e-9, None):
        assert gaussian_taps(s) == (1.0, 0.0)
    with pytest.raises(ValueError, match="3x3"):
        gaussian_taps(1.25)


def blur_cases(rs, n):
    shapes = [(1, 1), (1, 3), (3, 1), (2, 2), (1, 40), (40, 1), (2, 17), (480, 480)]
    for k in range(n):
        h, w = shapes[k] if k < len(shapes) else (int(rs.randint(1, 80)), int(rs.randint(1, 80)))
        sigma = float(rs.rand()) if k % 3 == 0 else 0.6061 + float(rs.rand()) * 0.39
        yield (rs.rand(h, w, 3) * 255).astype(np.float32), sigma


def test_gaussian_blur_restatement_against_cv2():
    """Bit-exact against cv2.GaussianBlur whenever cv2 runs its baseline (non-FMA) code: cv2.setUseOptimized(False), IPP
    on or off.  With the optimised dispatch (the default) the SIMD path fuses multiply-adds: the float results differ by a
    few ulps and, after np.uint8, a handful of pixels in a million move by one level."""
    cv2 = pytest.importorskip("cv2")
    had_ipp, had_opt = cv2.ipp.useIPP(), cv2.useOptimized()
    try:
        for ipp in (False, True):
            for opt in (False, True):
                cv2.ipp.setUseIPP(ipp)
                cv2.setUseOptimized(opt)
                rs = np.random.RandomState(15)
                exact, diff, n = 0, 0, 0
                cases = list(blur_cases(rs, 160))
                for img, sigma in cases:
                    k = vo.blur_ksize(sigma)
                    ref = cv2.GaussianBlur(img, (k, k), sigmaX=sigma, sigmaY=sigma, borderType=cv2.BORDER_REFLECT_101)
                    got = vo.cv_gaussian_blur_f32(img, sigma)
                    exact += np.array_equal(ref, got)
                    d = np.abs(np.uint8(ref).astype(int) - np.uint8(got).astype(int))
                    assert d.max() <= 1, (ipp, opt, img.shape, sigma)
                    diff += int((d > 0).sum())
                    n += d.size
                print(f"ipp={ipp} optimized={opt}: {exact}/{len(cases)} images bit-exact, uint8 differs at {diff}/{n}")
                if not opt:
                    assert exact == len(cases)
                else:
                    assert diff <= 1e-4 * n
    finally:
        cv2.ipp.setUseIPP(had_ipp)
        cv2.setUseOptimized(had_opt)


def test_val_tail_against_reference_goldens():
    """The reference as run: cv2.resize through the wheel's IPP float kernels (<= 3e-3 from OpenCV's own code before
    np.uint8), so labels are exact and images agree except a small fraction of pixels by one uint8 level."""
    g = np.load(GOLD)
    crop, mean, std = int(g["val_crop"]), g["mean"].tolist(), g["std"].tolist()
    one_level = 1.0 / 255.0 / min(std) * 1.001
    for i in range(int(g["n_val"])):
        x, y = vo.sample_val_tail(g[f"v{i}/image"], g[f"v{i}/label"], crop, mean, std)
        assert torch.equal(y, torch.from_numpy(g[f"v{i}/y"])), i
        d = (x - torch.from_numpy(g[f"v{i}/x"])).abs()
        assert d.max().item() <= one_level and (d > 0).float().mean().item() < 0.01, (i, d.max().item())
    assert (g["v0/label"] == -1).any() and (g["v0/y"] == -1).any() and (g["v0/y"] == 255).any()


def test_val_tail_bit_exact_with_opencvs_own_resize():
    """With IPP off, cv2.resize + PIL + the reference's crop arithmetic equal the restatement bit for bit."""
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    from oracle import data as od
    had = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        rs = np.random.RandomState(16)
        mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
        for k in range(30):
            H, W = int(rs.randint(5, 200)), int(rs.randint(5, 200))
            crop = int(rs.randint(1, 90))
            im = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
            lb = rs.randint(-1, 256, (H, W)).astype(np.int32)
            h, w = (crop, int(crop * W / H)) if H < W else (int(crop * H / W), crop)
            ri = cv2.resize(im.astype(np.float32), (w, h), interpolation=cv2.INTER_LINEAR)
            rl = np.asarray(Image.fromarray(lb).resize((w, h), resample=Image.NEAREST), dtype=np.int32)
            y0, x0 = (h - crop) // 2, (w - crop) // 2
            rx, ry = od.sample_tail(np.uint8(ri), rl, crop, y0, x0, False, mean, std)
            x, y = vo.sample_val_tail(im, lb, crop, mean, std)
            assert torch.equal(x, rx) and torch.equal(y, ry), (H, W, crop)
    finally:
        cv2.ipp.setUseIPP(had)


def test_val_geometry_is_the_reference_arithmetic():
    from seg_b200.data import val_geometry
    rs = np.random.RandomState(17)
    for _ in range(2000):
        h, w, crop = int(rs.randint(1, 3000)), int(rs.randint(1, 3000)), int(rs.randint(1, 1000))
        hh, ww = vo.val_size(h, w, crop)
        assert val_geometry(h, w, crop) == (hh, ww, (hh - crop) // 2, (ww - crop) // 2)
        assert min(hh, ww) == crop and max(hh, ww) >= crop
    assert val_geometry(1024, 2048, 480) == (480, 960, 0, 240)
    for crop in (None, 0):
        with pytest.raises(ValueError, match="crop_size"):
            val_geometry(10, 20, crop)


def test_blurred_chain_against_reference_goldens():
    """scale, rotate, pad, crop, flip, BLUR, np.uint8, ToTensor, Normalize against the reference's __getitem__ as run
    (IPP resize, optimised GaussianBlur): labels exact, images within one uint8 level on < 1 % of the pixels."""
    g = np.load(GOLD)
    crop, mean, std = int(g["crop"]), g["mean"].tolist(), g["std"].tolist()
    one_level = 1.0 / 255.0 / min(std) * 1.001
    bands = set()
    for i in range(int(g["n_train"])):
        h, w, angle, y0, x0, flip = (int(v) for v in g[f"t{i}/draw"])
        sigma = float(g[f"t{i}/sigma"])
        bands.add(vo.blur_ksize(sigma))
        x, y = vo.sample_blur_tail(g[f"t{i}/image"], g[f"t{i}/label"], h, w, crop, y0, x0, bool(flip), mean, std, angle, sigma)
        assert torch.equal(y, torch.from_numpy(g[f"t{i}/y"])), i
        d = (x - torch.from_numpy(g[f"t{i}/x"])).abs()
        assert d.max().item() <= one_level and (d > 0).float().mean().item() < 0.01, (i, d.max().item())
    assert bands == {1, 3}


def test_blur_draw_order_matches_reference():
    from seg_b200.data import draw_blur, draw_crop_flip, draw_rotate, draw_scale
    g = np.load(GOLD)
    crop, base = int(g["crop"]), int(g["base_size"])
    for i in range(int(g["n_train"])):
        h0, w0 = g[f"t{i}/image"].shape[:2]
        random.seed(500 + i)  # the seed the golden generator gave the reference's __getitem__
        h, w = draw_scale(h0, w0, base, scale=True)
        angle = draw_rotate(True)
        y0, x0, flip = draw_crop_flip(h, w, crop, flip=True)
        sigma = draw_blur(True)
        assert [h, w, angle, y0, x0, int(flip)] == [int(v) for v in g[f"t{i}/draw"]] and sigma == float(g[f"t{i}/sigma"]), i
    assert draw_blur(False) is None


def test_blur_commutes_with_the_flip():
    """The device kernel blurs the unflipped crop and flips the result; the reference flips, then blurs."""
    rs = np.random.RandomState(18)
    for img, sigma in blur_cases(rs, 40):
        a = vo.cv_gaussian_blur_f32(np.fliplr(img).copy(), sigma)
        b = np.fliplr(vo.cv_gaussian_blur_f32(img, sigma))
        assert np.array_equal(a.view(np.int32), np.ascontiguousarray(b).view(np.int32)), (img.shape, sigma)
    assert math.isclose(sum(float(t) for t in (vo.cv_gaussian_taps(0.8)[0], *2 * [vo.cv_gaussian_taps(0.8)[1]])), 1.0, rel_tol=1e-6)
