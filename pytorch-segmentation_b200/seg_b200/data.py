"""Input pipeline tail on the device (SURVEY.md §8f row 2).

The reference finishes every sample on a CPU worker — zero-pad to the crop size, random crop, random horizontal flip,
`ToTensor`, `Normalize`, label -> int64 (base/base_dataset.py:93-123,129-136) — and ships fp32 images + int64 labels over
PCIe (20 bytes per pixel) through `DataPrefetcher` (base/base_dataloader.py:49-85).  Here the scaled/rotated uint8 sample
crosses PCIe as it is (4 bytes per pixel with a uint8 label) and ONE kernel (`seg_augment_batch_u8`) performs the tail
for the whole batch, bit-exactly (same fp32 operations).  The random draws stay on the host, in the reference's order
(crop row, crop column, flip), so a seeded run is reproducible against the reference.

    DeviceBatcher(mean, std, crop_size, device)      — stage(samples) -> (images fp32 [B,3,crop,crop], labels int64 [B,crop,crop])
    DevicePrefetcher(loader, device, stop_after=None, batcher=None, val=False) — drop-in for the reference's DataPrefetcher;
        a loader that yields ready (float image batch, long label batch) pairs is passed through exactly as the reference
        does, a loader that yields lists of raw samples goes through the batcher (stage, or stage_val for a validation
        loader's raw (image, label) pairs when val=True).
"""
import math
import random

import numpy as np
import torch

from . import lib, ops

_ENTRY = np.dtype([("img_off", "<i8"), ("lbl_off", "<i8"), ("h", "<i4"), ("w", "<i4"), ("y0", "<i4"), ("x0", "<i4"),
                   ("flip", "<i4"), ("lbl_bytes", "<i4")])


_SCALE_ENTRY = np.dtype([("img_off", "<i8"), ("lbl_off", "<i8"), ("scale_x", "<f8"), ("scale_y", "<f8"), ("src_h", "<i4"),
                         ("src_w", "<i4"), ("h", "<i4"), ("w", "<i4"), ("y0", "<i4"), ("x0", "<i4"), ("flip", "<i4"), ("lbl_bytes", "<i4")])


_FULL_ENTRY = np.dtype([("img_off", "<i8"), ("lbl_off", "<i8"), ("scale_x", "<f8"), ("scale_y", "<f8"), ("a11", "<f8"), ("a12", "<f8"),
                        ("b1", "<f8"), ("a21", "<f8"), ("a22", "<f8"), ("b2", "<f8"), ("src_h", "<i4"), ("src_w", "<i4"), ("h", "<i4"),
                        ("w", "<i4"), ("y0", "<i4"), ("x0", "<i4"), ("flip", "<i4"), ("lbl_bytes", "<i4")])


def draw_rotate(rotate=True, rng=random):
    """The angle draw of base_dataset.py:78 (between the scale draw and the crop draws); None when rotation is off."""
    return rng.randint(-10, 10) if rotate else None


def inverse_rotation(w, h, angle):
    """(a11, a12, b1, a21, a22, b2): the inverse of cv2.getRotationMatrix2D((w/2, h/2), angle, 1.0) in float64, the operations
    cv::getRotationMatrix2D and cv::warpAffine perform (imgwarp.cpp) in their order; identity for angle None."""
    if angle is None:
        return 1.0, 0.0, 0.0, 0.0, 1.0, 0.0
    a = angle * (math.pi / 180.0)
    alpha, beta = math.cos(a) * 1.0, math.sin(a) * 1.0
    cx, cy = float(np.float32(w / 2)), float(np.float32(h / 2))  # Point2f
    m00, m01, m02 = alpha, beta, (1 - alpha) * cx - beta * cy
    m10, m11, m12 = -beta, alpha, beta * cx + (1 - alpha) * cy
    d = m00 * m11 - m01 * m10
    d = 1.0 / d if d != 0 else 0.0
    a11, a22, a12, a21 = m11 * d, m00 * d, -m01 * d, -m10 * d
    return a11, a12, -a11 * m02 - a12 * m12, a21, a22, -a21 * m02 - a22 * m12


def draw_blur(blur=True, rng=random):
    """The Gaussian-blur sigma of base_dataset.py:114-119 (drawn after the flip); None when blur is off."""
    return rng.random() if blur else None


def gaussian_taps(sigma):
    """(centre, side) float32 taps of cv2.GaussianBlur(image, (k, k), sigma, sigma) with the reference's kernel size
    k = int(3.3 * sigma) made odd: (1, 0) for k = 1 (no blur, also for sigma None), else getGaussianKernel(3, sigma, CV_32F)
    as OpenCV computes it (float64: t = exp(4 * (-0.125 / sigma^2)), normalised by 1 / (2t + 1), rounded to float32)."""
    if sigma is None:
        return 1.0, 0.0
    k = int(3.3 * sigma)
    k = k + 1 if k % 2 == 0 else k
    if k == 1:
        return 1.0, 0.0
    if k != 3:
        raise ValueError(f"blur: sigma {sigma} gives a {k}x{k} kernel; the device blur implements 3x3 (sigma < 1.2121...)")
    t = math.exp(4.0 * (-0.125 / (sigma * sigma)))
    mul = 1.0 / (t * 2.0 + 1.0)
    return float(np.float32(1.0 * mul)), float(np.float32(t * mul))


def val_geometry(h, w, crop_size):
    """(h', w', y0, x0) of _val_augmentation (base_dataset.py:40-61): the size whose short side is crop_size, in the
    reference's Python arithmetic, and the centre crop's origin."""
    if not crop_size:
        raise ValueError("validation tail: crop_size None / 0 means no resize and no crop (variable-size batches), which the "
                         "device tail does not build; set a crop_size")
    crop = int(crop_size)
    h2, w2 = (crop, int(crop * w / h)) if h < w else (int(crop * h / w), crop)
    return h2, w2, (h2 - crop) // 2, (w2 - crop) // 2


def pil_nearest_index(src, dst):
    """Source index per destination index of PIL's Image.resize(NEAREST) (Geometry.c ImagingScaleAffine): a float64
    coordinate that starts at a/2 and ACCUMULATES a = src / dst per pixel, truncated (np.add.accumulate adds in order)."""
    a = float(src) / dst
    xo = np.add.accumulate(np.concatenate([[0.0 + a * 0.5], np.full(dst - 1, a)]))
    idx = xo.astype(np.int64)
    assert idx.min() >= 0 and idx.max() < src
    return idx.astype(np.int32)


def draw_scale(h, w, base_size, scale=True, rng=random):
    """Size after the random-scale resize of base_dataset.py:66-72 (the long side becomes a draw in [0.5, 2] x base_size)."""
    if not base_size:
        return h, w
    longside = rng.randint(int(base_size * 0.5), int(base_size * 2.0)) if scale else base_size
    return (longside, int(1.0 * longside * w / h + 0.5)) if h > w else (int(1.0 * longside * h / w + 0.5), longside)


def draw_crop_flip(h, w, crop_size, flip=True, rng=random):
    """The draws of base_dataset.py:107-121 in the reference's order: crop origin in the padded image, then the flip."""
    ph, pw = max(h, crop_size), max(w, crop_size)
    y0 = rng.randint(0, ph - crop_size)
    x0 = rng.randint(0, pw - crop_size)
    f = bool(flip and rng.random() > 0.5)
    return y0, x0, f


def check_crop_origins(crop, dims):
    """dims: (h, w, y0, x0) per sample, h x w the image the crop is taken from.  The kernels trust the table, and a negative
    origin would read before the image, so an origin outside [0, max(h, crop) - crop] is refused before anything is staged."""
    for b, (h, w, y0, x0) in enumerate(dims):
        ym, xm = max(int(h), crop) - crop, max(int(w), crop) - crop
        if not (0 <= int(y0) <= ym and 0 <= int(x0) <= xm):
            raise ValueError(f"DeviceBatcher: sample {b}: crop origin (y0={y0}, x0={x0}) outside [0, {ym}] x [0, {xm}] "
                             f"for a {h} x {w} image and crop {crop}")


class DeviceBatcher:
    def __init__(self, mean, std, crop_size, device, max_bytes=64 << 20):
        assert _ENTRY.itemsize == lib.load().seg_aug_entry_bytes()
        if not crop_size:
            raise ValueError("DeviceBatcher: crop_size None / 0 means the reference neither pads nor crops (and its validation "
                             "tail does not resize), so batches would have variable sizes; the device tails need a crop_size")
        self.mean, self.std = [float(v) for v in mean], [float(v) for v in std]
        self.crop = int(crop_size)
        self.device = torch.device(device)
        self.capacity = int(max_bytes)
        self._host = [torch.empty(self.capacity, dtype=torch.uint8).pin_memory() for _ in range(2)]  # double-buffered staging
        self._slot = 0
        self._events = [None, None]

    def stage(self, samples):
        """samples: sequence of (image uint8 [h,w,3], label uint8|int32 [h,w] or None, y0, x0, flip).  Packs them into
        pinned memory, copies once, launches the kernel on the current stream.  Returns (images, labels)."""
        B = len(samples)
        check_crop_origins(self.crop, [(np.shape(s[0])[0], np.shape(s[0])[1], s[2], s[3]) for s in samples])
        slot = self._slot
        self._slot ^= 1
        if self._events[slot] is not None:
            self._events[slot].synchronize()  # the previous H2D copy out of this staging buffer has finished
        host = self._host[slot].numpy()
        table = np.zeros(B, dtype=_ENTRY)
        off = B * _ENTRY.itemsize
        want_labels = samples[0][1] is not None
        for b, (img, lbl, y0, x0, flip) in enumerate(samples):
            img = np.ascontiguousarray(img, dtype=np.uint8)
            h, w = img.shape[:2]
            assert img.shape == (h, w, 3), "images are HWC uint8 with 3 channels"
            n = img.size
            lb, lbl_off = 1, -1
            if lbl is not None:
                lbl = np.ascontiguousarray(lbl)
                assert lbl.shape == (h, w) and lbl.dtype in (np.uint8, np.int32), "labels are uint8 or int32 [h,w]"
                lb = lbl.dtype.itemsize
            need = off + n + 8 + (h * w * lb if lbl is not None else 0)
            if need > self.capacity:
                raise RuntimeError(f"DeviceBatcher: batch needs more than max_bytes={self.capacity} of staging memory")
            host[off:off + n] = img.reshape(-1)
            img_off = off
            off += (n + 3) // 4 * 4  # keep int32 label maps 4-byte aligned
            if lbl is not None:
                nb = h * w * lb
                host[off:off + nb] = lbl.reshape(-1).view(np.uint8)
                lbl_off = off
                off += (nb + 3) // 4 * 4
            table[b] = (img_off, lbl_off, h, w, int(y0), int(x0), int(bool(flip)), lb)
        host[:B * _ENTRY.itemsize] = table.view(np.uint8)
        self.last_staged_bytes = off
        dev = self._host[slot][:off].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        tab = dev[:B * _ENTRY.itemsize]
        return ops.augment_batch_u8(dev, tab, B, self.crop, self.crop, self.mean, self.std, want_labels=want_labels)

    def _stage_raw(self, samples, dtype, record, head=None, tail=None):
        """Packs RAW samples (image uint8 [H,W,3], label uint8|int32 [H,W] or None, ...) into the pinned staging buffer and
        copies it to the device once: the B `dtype` records first, then `head` (a float32 array, e.g. per-sample blur taps),
        then every image and label map 4-byte aligned, each label map followed by `tail(b, H, W)` (an int32 array) when given.
        record(b, img_off, lbl_off, H, W, lbl_bytes) -> the record of sample b.  Returns (device arena, head offset)."""
        B = len(samples)
        slot = self._slot
        self._slot ^= 1
        if self._events[slot] is not None:
            self._events[slot].synchronize()
        host = self._host[slot].numpy()
        table = np.zeros(B, dtype=dtype)
        head_off = off = B * dtype.itemsize
        if head is not None:
            head = np.ascontiguousarray(head, dtype=np.float32)
            host[off:off + head.nbytes] = head.reshape(-1).view(np.uint8)
            off += head.nbytes
        for b, s in enumerate(samples):
            img, lbl = np.ascontiguousarray(s[0], dtype=np.uint8), s[1]
            H, W = img.shape[:2]
            assert img.shape == (H, W, 3), "images are HWC uint8 with 3 channels"
            n = img.size
            lb, lbl_off, extra = 1, -1, None
            if lbl is not None:
                lbl = np.ascontiguousarray(lbl)
                assert lbl.shape == (H, W) and lbl.dtype in (np.uint8, np.int32), "labels are uint8 or int32 [H,W]"
                lb = lbl.dtype.itemsize
                extra = tail(b, H, W) if tail is not None else None
            need = off + n + 8 + (H * W * lb if lbl is not None else 0) + (extra.nbytes if extra is not None else 0)
            if need > self.capacity:
                raise RuntimeError(f"DeviceBatcher: batch needs more than max_bytes={self.capacity} of staging memory")
            host[off:off + n] = img.reshape(-1)
            img_off = off
            off += (n + 3) // 4 * 4
            if lbl is not None:
                nb = H * W * lb
                host[off:off + nb] = lbl.reshape(-1).view(np.uint8)
                lbl_off = off
                off += (nb + 3) // 4 * 4
                if extra is not None:
                    host[off:off + extra.nbytes] = np.ascontiguousarray(extra, dtype=np.int32).view(np.uint8)
                    off += extra.nbytes
            table[b] = record(b, img_off, lbl_off, H, W, lb)
        host[:B * dtype.itemsize] = table.view(np.uint8)
        self.last_staged_bytes = off
        dev = self._host[slot][:off].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        return dev, head_off

    def stage_scaled(self, samples):
        """samples: sequence of (RAW image uint8 [H,W,3], RAW label uint8|int32 [H,W] or None, h, w, y0, x0, flip): the sample
        is resized to h x w (cv2.resize arithmetic, base_dataset.py:66-75) and then padded / cropped / flipped / normalised
        — in one kernel, without a resized intermediate (`seg_augment_scale_batch_u8`)."""
        assert _SCALE_ENTRY.itemsize == lib.load().seg_aug_scale_entry_bytes()
        B = len(samples)
        check_crop_origins(self.crop, [(s[2], s[3], s[4], s[5]) for s in samples])

        def record(b, img_off, lbl_off, H, W, lb):
            _, _, h, w, y0, x0, flip = samples[b]
            # cv::resize: inv_scale = dsize / ssize, scale = 1. / inv_scale — float64, computed here so the kernel sees the same bits
            return (img_off, lbl_off, 1.0 / (int(w) / W), 1.0 / (int(h) / H), H, W, int(h), int(w), int(y0), int(x0), int(bool(flip)), lb)

        dev, _ = self._stage_raw(samples, _SCALE_ENTRY, record)
        return ops.augment_scale_batch_u8(dev, dev[:B * _SCALE_ENTRY.itemsize], B, self.crop, self.crop, self.mean, self.std,
                                          want_labels=samples[0][1] is not None)

    def stage_full(self, samples, sigmas=None):
        """(bit-exact against the staged oracle, tests/test_data_tail_gpu.py.)  samples: sequence of
        (RAW image, RAW label or None, h, w, angle or None, y0, x0, flip): resize to h x w, rotate by `angle` degrees about the
        centre (base_dataset.py:77-83), pad / crop / flip / normalise — one kernel (`seg_augment_full_batch_u8`).
        sigmas: per-sample Gaussian blur sigma or None (draw_blur; base_dataset.py:114-119), applied after the flip; when any
        sample's kernel size is 3 the batch runs `seg_augment_full_blur_batch_u8`, whose k = 1 samples are bit-identical
        to the unblurred kernel's."""
        assert _FULL_ENTRY.itemsize == lib.load().seg_aug_full_entry_bytes()
        B = len(samples)
        check_crop_origins(self.crop, [(s[2], s[3], s[5], s[6]) for s in samples])
        taps = None
        if sigmas is not None:
            if len(sigmas) != B:
                raise ValueError(f"DeviceBatcher: {len(sigmas)} blur sigmas for {B} samples")
            taps = np.array([gaussian_taps(s) for s in sigmas], dtype=np.float32)
            if (taps[:, 1] == 0).all():
                taps = None  # nothing to blur: the unblurred kernel gives the same bytes

        def record(b, img_off, lbl_off, H, W, lb):
            _, _, h, w, angle, y0, x0, flip = samples[b]
            return (img_off, lbl_off, 1.0 / (int(w) / W), 1.0 / (int(h) / H)) + inverse_rotation(int(w), int(h), angle) + \
                (H, W, int(h), int(w), int(y0), int(x0), int(bool(flip)), lb)

        dev, head_off = self._stage_raw(samples, _FULL_ENTRY, record, head=taps)
        tab, want_labels = dev[:B * _FULL_ENTRY.itemsize], samples[0][1] is not None
        if taps is None:
            return ops.augment_full_batch_u8(dev, tab, B, self.crop, self.crop, self.mean, self.std, want_labels=want_labels)
        dtaps = dev[head_off:head_off + taps.nbytes].view(torch.float32)
        return ops.augment_full_blur_batch_u8(dev, tab, dtaps, B, self.crop, self.crop, self.mean, self.std, want_labels=want_labels)

    def stage_val(self, samples):
        """The validation tail of base_dataset.py:40-61 and :129-136.  samples: sequence of (RAW image uint8 [H,W,3], RAW label
        uint8|int32 [H,W] or None).  Each sample is resized so that its short side is crop_size (cv2.resize INTER_LINEAR on
        the image, PIL's NEAREST on the label, negative labels kept), centre-cropped, truncated to uint8 and normalised — one
        kernel (`seg_augment_val_batch_u8`), no resized intermediate."""
        assert _SCALE_ENTRY.itemsize == lib.load().seg_aug_scale_entry_bytes()
        B = len(samples)
        for b, s in enumerate(samples):
            if len(s) != 2:
                raise ValueError(f"DeviceBatcher.stage_val: sample {b} is not an (image, label) pair")
            im, lb = s
            if np.ndim(im) != 3 or np.shape(im)[2] != 3 or min(np.shape(im)[:2]) < 1:
                raise ValueError(f"DeviceBatcher.stage_val: sample {b}: image of shape {np.shape(im)} is not [H, W, 3]")
            if lb is not None and tuple(np.shape(lb)) != tuple(np.shape(im)[:2]):
                raise ValueError(f"DeviceBatcher.stage_val: sample {b}: label of shape {np.shape(lb)} for a {np.shape(im)} image")
            if (lb is None) != (samples[0][1] is None):
                raise ValueError("DeviceBatcher.stage_val: either every sample has a label or none has")
        geom = [val_geometry(np.shape(s[0])[0], np.shape(s[0])[1], self.crop) for s in samples]
        check_crop_origins(self.crop, [(h, w, y0, x0) for h, w, y0, x0 in geom])

        def record(b, img_off, lbl_off, H, W, lb):
            h, w, y0, x0 = geom[b]
            return (img_off, lbl_off, 1.0 / (w / W), 1.0 / (h / H), H, W, h, w, y0, x0, 0, lb)

        def tables(b, H, W):
            h, w = geom[b][:2]
            return np.concatenate([pil_nearest_index(W, w), pil_nearest_index(H, h)])

        dev, _ = self._stage_raw(samples, _SCALE_ENTRY, record, tail=tables)
        return ops.augment_val_batch_u8(dev, dev[:B * _SCALE_ENTRY.itemsize], B, self.crop, self.crop, self.mean, self.std,
                                        want_labels=samples[0][1] is not None)

    def stage_random(self, raw, flip=True, rng=random):
        """raw: sequence of (image, label).  Draws crop origin / flip per sample like the reference's worker would."""
        return self.stage([(im, lb) + draw_crop_flip(im.shape[0], im.shape[1], self.crop, flip, rng) for im, lb in raw])


class DevicePrefetcher:
    """base/base_dataloader.py:49-85 with the same protocol (`len`, iteration yields (input, target) on the device, the
    next batch is staged on a side stream while the current one is consumed, `stop_after`)."""

    def __init__(self, loader, device, stop_after=None, batcher=None, val=False):
        self.loader = loader
        self.val = val  # raw batches are (image, label) pairs of a validation loader: batcher.stage_val
        self.dataset = getattr(loader, "dataset", None)
        self.stream = torch.cuda.Stream()
        self.stop_after = stop_after
        self.next_input = None
        self.next_target = None
        self.device = device
        self.batcher = batcher

    def __len__(self):
        return len(self.loader)

    def preload(self):
        try:
            item = next(self.loaditer)
        except StopIteration:
            self.next_input = None
            self.next_target = None
            return
        with torch.cuda.stream(self.stream):
            if isinstance(item, (tuple, list)) and len(item) == 2 and isinstance(item[0], torch.Tensor) and item[0].is_floating_point():
                self.next_input = item[0].cuda(device=self.device, non_blocking=True)   # the reference's path, unchanged
                self.next_target = item[1].cuda(device=self.device, non_blocking=True)
            else:
                if self.batcher is None:
                    raise RuntimeError("DevicePrefetcher: the loader yields raw uint8 samples but no DeviceBatcher was given")
                self.next_input, self.next_target = (self.batcher.stage_val if self.val else self.batcher.stage)(item)

    def __iter__(self):
        count = 0
        self.loaditer = iter(self.loader)
        self.preload()
        while self.next_input is not None:
            torch.cuda.current_stream().wait_stream(self.stream)
            input, target = self.next_input, self.next_target
            input.record_stream(torch.cuda.current_stream())
            if target is not None:
                target.record_stream(torch.cuda.current_stream())
            self.preload()
            count += 1
            yield input, target
            if type(self.stop_after) is int and (count > self.stop_after):
                break
