"""CPU restatement of the two parts of the reference's sample pipeline that the device tails gained last: the validation
tail (base/base_dataset.py:40-61, then :129-136) and the Gaussian blur of the training tail (:114-119).  TEST
INFRASTRUCTURE ONLY, built on oracle/data.py's restatements of cv2.resize / warpAffine and of the ToTensor / Normalize tail.
Pinned to cv2 / PIL by tests/test_val_blur_oracle_cpu.py and to the reference's own BaseDataSet.__getitem__ by
tests/golden/data_val_blur.npz (tools/make_golden_val_blur.py)."""
import math

import numpy as np
import torch

from oracle import data as od


def pil_resize_nearest(lbl, w, h):
    """np.asarray(Image.fromarray(lbl).resize((w, h), Image.NEAREST)) for an int32 (mode "I") or uint8 (mode "L") map.
    Pillow (Geometry.c ImagingScaleAffine) starts the float64 source coordinate at a/2 with a = src / dst and ADDS a once
    per destination pixel, truncating each partial sum; the accumulated rounding makes some indices differ from
    floor((d + 0.5) * a), so the sums are replayed in order here (np.add.accumulate is sequential)."""
    def index(src, dst):
        a = float(src) / dst
        return np.add.accumulate(np.concatenate([[0.0 + a * 0.5], np.full(dst - 1, a)])).astype(np.int64)
    sh, sw = lbl.shape[:2]
    if (sh, sw) == (h, w):
        return lbl.copy()
    return lbl[index(sh, h)][:, index(sw, w)]


def val_size(h, w, crop):
    """base_dataset.py:43-48: the short side becomes crop (Python float arithmetic, truncated)."""
    return (crop, int(crop * w / h)) if h < w else (int(crop * h / w), crop)


def sample_val_tail(image, label, crop, mean, std):
    """_val_augmentation + __getitem__: cv2.resize INTER_LINEAR (OpenCV's own float path) of the image, PIL NEAREST of
    the label, centre crop, np.uint8, ToTensor, Normalize, label -> int64.  label None: (x, None)."""
    H, W = image.shape[:2]
    h, w = val_size(H, W, crop)
    img = od.cv_resize_linear_f32(image, w, h)
    lab = pil_resize_nearest(np.asarray(label), w, h) if label is not None else np.zeros((h, w), np.int32)
    y0, x0 = (h - crop) // 2, (w - crop) // 2
    x, y = od.sample_tail(np.uint8(img), lab, crop, y0, x0, False, mean, std)
    return x, (y if label is not None else None)


def cv_gaussian_taps(sigma):
    """cv::getGaussianKernel(3, sigma, CV_32F) (smooth.dispatch.cpp, getGaussianKernelBitExact): float64
    t = exp((x*x) * (-0.125 / sigma^2)) with x*x = 4, sum = 2t + 1, taps t / sum and 1 / sum rounded to float32.
    Returns (centre, side)."""
    t = math.exp(4.0 * (-0.125 / (sigma * sigma)))
    mul = 1.0 / (t * 2.0 + 1.0)
    return np.float32(1.0 * mul), np.float32(t * mul)


def blur_ksize(sigma):
    """base_dataset.py:116-117"""
    k = int(3.3 * sigma)
    return k + 1 if k % 2 == 0 else k


def cv_gaussian_blur_f32(img, sigma):
    """cv2.GaussianBlur(img, (k, k), sigma, sigma, borderType=BORDER_REFLECT_101) for a float32 [h, w, c] image with the
    reference's k = blur_ksize(sigma) in {1, 3}.  k = 1 is a copy.  k = 3 is OpenCV's separable float filter
    (filter.simd.hpp SymmRowSmallFilter then SymmColumnSmallFilter): row R = S*k0 + (S[x-1] + S[x+1])*k1, column
    (R[y-1] + R[y+1])*k1 + R*k0, float32, each product and sum rounded (no fma); reflect-101 borders; an axis of length 1
    is not filtered.  Bit-exact against cv2 with cv2.setUseOptimized(False) (IPP on or off); with the optimised (AVX2 +
    FMA) dispatch cv2 fuses multiply-adds and differs by a few float32 ulps (tests/test_val_blur_oracle_cpu.py counts the
    uint8 pixels that changes)."""
    k = blur_ksize(sigma)
    assert k in (1, 3), k
    img = np.asarray(img, dtype=np.float32)
    if k == 1:
        return img.copy()
    k0, k1 = cv_gaussian_taps(sigma)

    def refl(n):
        i = np.arange(-1, n + 1)
        return np.where(i < 0, -i, np.where(i >= n, 2 * n - 2 - i, i))

    h, w = img.shape[:2]
    out = img
    if w > 1:
        S = out[:, refl(w)]
        out = (S[:, 1:-1] * k0 + (S[:, :-2] + S[:, 2:]) * k1).astype(np.float32)
    if h > 1:
        R = out[refl(h)]
        out = ((R[:-2] + R[2:]) * k1 + R[1:-1] * k0).astype(np.float32)
    return out


def sample_blur_tail(image, label, h, w, crop, y0, x0, flip, mean, std, angle=None, sigma=None):
    """base_dataset.py:66-136 staged as the reference runs it: resize to h x w, rotate by `angle`, zero-pad to the crop,
    crop at (y0, x0), flip, Gaussian blur of the FLOAT crop (sigma None: off), np.uint8, ToTensor, Normalize.
    crop: an int, or (crop_h, crop_w) for the device kernels' rectangular crops."""
    ch, cw = (crop, crop) if np.isscalar(crop) else crop
    img = od.cv_resize_linear_f32(image, w, h)
    lab = od.cv_resize_nearest(np.asarray(label), w, h)
    if angle is not None:
        M = od.cv_rotation_matrix((w / 2, h / 2), angle, 1.0)
        img = od.cv_warp_affine(img, M, w, h, linear=True)
        lab = od.cv_warp_affine(lab, M, w, h, linear=False)
    ph, pw = max(ch - h, 0), max(cw - w, 0)
    img = np.pad(img, ((0, ph), (0, pw), (0, 0)))[y0:y0 + ch, x0:x0 + cw]
    lab = np.pad(lab, ((0, ph), (0, pw)))[y0:y0 + ch, x0:x0 + cw]
    if flip:
        img, lab = np.fliplr(img).copy(), np.fliplr(lab).copy()
    if sigma is not None:
        img = cv_gaussian_blur_f32(img, sigma)
    if ch == cw:
        return od.sample_tail(np.uint8(img), lab, ch, 0, 0, False, mean, std)
    y = torch.from_numpy(np.array(lab, dtype=np.int32)).long()
    x = torch.from_numpy(np.ascontiguousarray(np.uint8(img))).permute(2, 0, 1).contiguous().to(torch.float32).div(255)  # ToTensor
    m, s = (torch.as_tensor(v, dtype=torch.float32).view(-1, 1, 1) for v in (mean, std))
    return x.sub_(m).div_(s), y  # Normalize
