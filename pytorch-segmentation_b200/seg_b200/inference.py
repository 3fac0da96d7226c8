"""Test-time augmentation of the reference's inference.py on the device (SURVEY.md §8f row 3).

    multi_scale_predict(model, image, scales, num_classes, device=None, flip=False)   — inference.py:58-79
    sliding_predict(model, image, num_classes, flip=True)                             — inference.py:26-56
    predict_labels(scores)                                                            — inference.py:156

Same signatures and arithmetic; what changes is where it runs.  The reference round-trips every scale through the host
(`ndimage.zoom` on a numpy copy, `model(...).cpu()`, `nn.Upsample` on the CPU, float64 numpy accumulation); here the
image pyramid, the flips, the up-sampling back to the input size and the accumulation are the fp32 kernels of
`seg_data.cu` and nothing leaves the GPU until the caller asks for the label map.  `ndimage.zoom(order=1)` with the
default `grid_mode=False` maps output pixel o to input o*(in-1)/(out-1) in float64 (bilinear with align_corners=True),
rounds the output size with Python's round(), and — mode='constant' — writes 0 where that coordinate rounds past the last
input sample (for some size pairs the last row / column of a zoomed image is black in the reference): all reproduced
(`seg_resize_nchw_f32` mode 2).  Returns a device tensor [num_classes, H, W] (the
reference returns the same values as a float64 numpy array).
"""
from math import ceil

import numpy as np
import torch

from . import ops


def _require_cuda(image):
    if not image.is_cuda:
        raise RuntimeError("seg_b200.inference runs on an H100 only; there is no CPU fallback")


def multi_scale_predict(model, image, scales, num_classes, device=None, flip=False):
    _require_cuda(image)
    image = image.detach().contiguous().float()
    N, _, H, W = image.shape
    assert N == 1, "inference.py feeds one image at a time (squeeze(0) at inference.py:76)"
    total = torch.zeros((1, num_classes, H, W), dtype=torch.float32, device=image.device)
    w = 1.0 / len(scales)
    with torch.no_grad():
        for scale in scales:
            Hs, Ws = int(round(H * float(scale))), int(round(W * float(scale)))
            scaled = image if (Hs, Ws) == (H, W) else ops.resize_nchw(image, Hs, Ws, zoom=True)
            pred = model(scaled).contiguous().float()
            if flip:
                flipped = ops.resize_nchw(scaled, Hs, Ws, align_corners=True, flip_x=True)  # same size: an exact flip
                pred_f = model(flipped).contiguous().float()
                # 0.5 * (upsample(pred_f).flip(-1) + upsample(pred))  accumulated with weight 1/len(scales)
                ops.resize_nchw(pred, H, W, align_corners=True, alpha=0.5 * w, out=total, beta=1.0)
                ops.resize_nchw(pred_f, H, W, align_corners=True, flip_x=True, alpha=0.5 * w, out=total, beta=1.0)
            else:
                ops.resize_nchw(pred, H, W, align_corners=True, alpha=w, out=total, beta=1.0)
    return total[0]


def pad_image(img, target_size):
    """inference.py:20-24: zero-pad bottom / right up to target_size."""
    rows, cols = max(target_size[0] - img.shape[2], 0), max(target_size[1] - img.shape[3], 0)
    if rows == 0 and cols == 0:
        return img.contiguous()
    out = torch.zeros((img.shape[0], img.shape[1], img.shape[2] + rows, img.shape[3] + cols), dtype=img.dtype, device=img.device)
    ops.window_add_nchw(img.contiguous(), out, 0, 0, img.shape[2], img.shape[3])
    return out


def sliding_windows(H, W):
    """Tile geometry of inference.py:27-35: tile = size // 2.5, overlap 1/3, one stride (from the tile HEIGHT) for both axes."""
    tile = (int(H // 2.5), int(W // 2.5))
    stride = ceil(tile[0] * (1 - 1 / 3))
    rows = int(ceil((H - tile[0]) / stride) + 1)
    cols = int(ceil((W - tile[1]) / stride) + 1)
    wins = []
    for r in range(rows):
        for c in range(cols):
            x_min, y_min = int(c * stride), int(r * stride)
            wins.append((y_min, min(y_min + tile[0], H), x_min, min(x_min + tile[1], W)))
    return tile, wins


def sliding_predict(model, image, num_classes, flip=True):
    _require_cuda(image)
    image = image.detach().contiguous().float()
    N, _, H, W = image.shape
    assert N == 1, "inference.py feeds one image at a time (squeeze(0) at inference.py:53)"
    tile, wins = sliding_windows(H, W)
    total = torch.zeros((1, num_classes, H, W), dtype=torch.float32, device=image.device)
    count = np.zeros((H, W), dtype=np.float32)
    with torch.no_grad():
        for (y0, y1, x0, x1) in wins:
            if y1 <= y0 or x1 <= x0:
                # an empty window (portrait images: the one stride, from the tile height, can start a column at or past
                # the right edge); the reference predicts on a padded empty tile and adds nothing from it
                continue
            padded = pad_image(image[:, :, y0:y1, x0:x1], tile)
            pred = model(padded).contiguous().float()
            h, w = y1 - y0, x1 - x0
            if flip:
                flipped = ops.resize_nchw(padded, padded.shape[2], padded.shape[3], align_corners=True, flip_x=True)
                pred_f = model(flipped).contiguous().float()
                ops.window_add_nchw(pred, total, y0, x0, h, w, alpha=0.5)
                ops.window_add_nchw(pred_f, total, y0, x0, h, w, flip_x=True, alpha=0.5)
            else:
                ops.window_add_nchw(pred, total, y0, x0, h, w)
            count[y0:y1, x0:x1] += 1
    ops.div_by_count_nchw(total, torch.from_numpy(count).to(image.device))
    return total[0]


def predict_labels(scores):
    """Label map of inference.py:156 (`softmax(dim=0).argmax(0)`) as an int64 device tensor: 0 where a pixel's scores hold
    a NaN or +inf (the reference's softmax column is then all NaN), elsewhere the first maximum score.  Pixels that no
    sliding window covers hold NaN scores (0 / 0, as in the reference) and get label 0."""
    s = scores if scores.dim() == 4 else scores.unsqueeze(0)
    _require_cuda(s)
    lab = ops.argmax_nchw(s.contiguous().float())
    return lab if scores.dim() == 4 else lab[0]
