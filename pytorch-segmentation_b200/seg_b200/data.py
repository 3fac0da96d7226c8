"""Input pipeline tail on the device (SURVEY.md §8f row 2).

The reference finishes every sample on a CPU worker — zero-pad to the crop size, random crop, random horizontal flip,
`ToTensor`, `Normalize`, label -> int64 (base/base_dataset.py:93-123,129-136) — and ships fp32 images + int64 labels over
PCIe (20 bytes per pixel) through `DataPrefetcher` (base/base_dataloader.py:49-85).  Here the scaled/rotated uint8 sample
crosses PCIe as it is (4 bytes per pixel with a uint8 label) and ONE kernel (`seg_augment_batch_u8`) performs the tail
for the whole batch, bit-exactly (same fp32 operations).  The random draws stay on the host, in the reference's order
(crop row, crop column, flip), so a seeded run is reproducible against the reference.

    DeviceBatcher(mean, std, crop_size, device)      — stage(samples) -> (images fp32 [B,3,crop,crop], labels int64 [B,crop,crop])
    DevicePrefetcher(loader, device, stop_after=None, batcher=None) — drop-in for the reference's DataPrefetcher;
        a loader that yields ready (float image batch, long label batch) pairs is passed through exactly as the reference
        does, a loader that yields lists of raw samples goes through the batcher.
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

    def stage_scaled(self, samples):
        """samples: sequence of (RAW image uint8 [H,W,3], RAW label uint8|int32 [H,W] or None, h, w, y0, x0, flip): the sample
        is resized to h x w (cv2.resize arithmetic, base_dataset.py:66-75) and then padded / cropped / flipped / normalised
        — in one kernel, without a resized intermediate (`seg_augment_scale_batch_u8`)."""
        assert _SCALE_ENTRY.itemsize == lib.load().seg_aug_scale_entry_bytes()
        B = len(samples)
        check_crop_origins(self.crop, [(s[2], s[3], s[4], s[5]) for s in samples])
        slot = self._slot
        self._slot ^= 1
        if self._events[slot] is not None:
            self._events[slot].synchronize()
        host = self._host[slot].numpy()
        table = np.zeros(B, dtype=_SCALE_ENTRY)
        off = B * _SCALE_ENTRY.itemsize
        want_labels = samples[0][1] is not None
        for b, (img, lbl, h, w, y0, x0, flip) in enumerate(samples):
            img = np.ascontiguousarray(img, dtype=np.uint8)
            H, W = img.shape[:2]
            assert img.shape == (H, W, 3), "images are HWC uint8 with 3 channels"
            n = img.size
            lb, lbl_off = 1, -1
            if lbl is not None:
                lbl = np.ascontiguousarray(lbl)
                assert lbl.shape == (H, W) and lbl.dtype in (np.uint8, np.int32), "labels are uint8 or int32 [H,W]"
                lb = lbl.dtype.itemsize
            if off + n + 8 + (H * W * lb if lbl is not None else 0) > self.capacity:
                raise RuntimeError(f"DeviceBatcher: batch needs more than max_bytes={self.capacity} of staging memory")
            host[off:off + n] = img.reshape(-1)
            img_off = off
            off += (n + 3) // 4 * 4
            if lbl is not None:
                nb = H * W * lb
                host[off:off + nb] = lbl.reshape(-1).view(np.uint8)
                lbl_off = off
                off += (nb + 3) // 4 * 4
            # cv::resize: inv_scale = dsize / ssize, scale = 1. / inv_scale — float64, computed here so the kernel sees the same bits
            table[b] = (img_off, lbl_off, 1.0 / (int(w) / W), 1.0 / (int(h) / H), H, W, int(h), int(w), int(y0), int(x0), int(bool(flip)), lb)
        host[:B * _SCALE_ENTRY.itemsize] = table.view(np.uint8)
        self.last_staged_bytes = off
        dev = self._host[slot][:off].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        return ops.augment_scale_batch_u8(dev, dev[:B * _SCALE_ENTRY.itemsize], B, self.crop, self.crop, self.mean, self.std,
                                          want_labels=want_labels)

    def stage_full(self, samples):
        """(bit-exact against the staged oracle, tests/test_data_tail_gpu.py.)  samples: sequence of
        (RAW image, RAW label or None, h, w, angle or None, y0, x0, flip): resize to h x w, rotate by `angle` degrees about the
        centre (base_dataset.py:77-83), pad / crop / flip / normalise — one kernel (`seg_augment_full_batch_u8`)."""
        assert _FULL_ENTRY.itemsize == lib.load().seg_aug_full_entry_bytes()
        B = len(samples)
        check_crop_origins(self.crop, [(s[2], s[3], s[5], s[6]) for s in samples])
        slot = self._slot
        self._slot ^= 1
        if self._events[slot] is not None:
            self._events[slot].synchronize()
        host = self._host[slot].numpy()
        table = np.zeros(B, dtype=_FULL_ENTRY)
        off = B * _FULL_ENTRY.itemsize
        want_labels = samples[0][1] is not None
        for b, (img, lbl, h, w, angle, y0, x0, flip) in enumerate(samples):
            img = np.ascontiguousarray(img, dtype=np.uint8)
            H, W = img.shape[:2]
            assert img.shape == (H, W, 3), "images are HWC uint8 with 3 channels"
            n = img.size
            lb, lbl_off = 1, -1
            if lbl is not None:
                lbl = np.ascontiguousarray(lbl)
                assert lbl.shape == (H, W) and lbl.dtype in (np.uint8, np.int32), "labels are uint8 or int32 [H,W]"
                lb = lbl.dtype.itemsize
            if off + n + 8 + (H * W * lb if lbl is not None else 0) > self.capacity:
                raise RuntimeError(f"DeviceBatcher: batch needs more than max_bytes={self.capacity} of staging memory")
            host[off:off + n] = img.reshape(-1)
            img_off = off
            off += (n + 3) // 4 * 4
            if lbl is not None:
                nb = H * W * lb
                host[off:off + nb] = lbl.reshape(-1).view(np.uint8)
                lbl_off = off
                off += (nb + 3) // 4 * 4
            table[b] = (img_off, lbl_off, 1.0 / (int(w) / W), 1.0 / (int(h) / H)) + inverse_rotation(int(w), int(h), angle) + \
                       (H, W, int(h), int(w), int(y0), int(x0), int(bool(flip)), lb)
        host[:B * _FULL_ENTRY.itemsize] = table.view(np.uint8)
        self.last_staged_bytes = off
        dev = self._host[slot][:off].to(self.device, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._events[slot] = ev
        return ops.augment_full_batch_u8(dev, dev[:B * _FULL_ENTRY.itemsize], B, self.crop, self.crop, self.mean, self.std,
                                         want_labels=want_labels)

    def stage_random(self, raw, flip=True, rng=random):
        """raw: sequence of (image, label).  Draws crop origin / flip per sample like the reference's worker would."""
        return self.stage([(im, lb) + draw_crop_flip(im.shape[0], im.shape[1], self.crop, flip, rng) for im, lb in raw])


class DevicePrefetcher:
    """base/base_dataloader.py:49-85 with the same protocol (`len`, iteration yields (input, target) on the device, the
    next batch is staged on a side stream while the current one is consumed, `stop_after`)."""

    def __init__(self, loader, device, stop_after=None, batcher=None):
        self.loader = loader
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
                self.next_input, self.next_target = self.batcher.stage(item)

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
