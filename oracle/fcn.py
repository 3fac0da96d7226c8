"""FCN8 (models/fcn.py:9-103) for the CPU oracle (TEST INFRASTRUCTURE — see oracle/__init__.py): a deterministic state_dict
factory with the reference's names and shapes, and a functional fp32 restatement of the forward pass.

  fcn8_forward -> fcn.py:76-97 (FCN8.forward): torchvision vgg16's features with features[0].padding = 100 and every
                  MaxPool2d in ceil mode, split at 17 / 24 (pool3 / pool4 / pool5); conv6 (7x7) ReLU conv7 ReLU score conv
                  (dropout not modelled: the train parity runs it at p = 0); three ConvTranspose2d upsamplings with the
                  scaled adj_pool4 / adj_pool3 skips cropped at 5 and 9 and the logits cropped at 31
"""
import numpy as np
import torch
import torch.nn.functional as F

from .models import _conv
from .weights import _Gen

VGG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")
SPLITS = (("pool3", 0), ("pool4", 17), ("pool5", 24))  # vgg16().features[:17], [17:24], [24:]
UPSAMPLERS = (("up_output", 4), ("up_pool4_out", 4), ("up_final", 16))


def _features():
    """[(feature index, stage, index in the stage, cin, cout or None for a pool)] of vgg16().features."""
    out, fi, cin = [], 0, 3
    for v in VGG:
        stage, base = [s for s in SPLITS if s[1] <= fi][-1]
        if v == "M":
            out.append((fi, stage, fi - base, cin, None))
            fi += 1
        else:
            out.append((fi, stage, fi - base, cin, v))
            cin = v
            fi += 2  # conv, ReLU
    return out


def upsampling_weight(c, k):
    """utils/helpers.py:get_upsampling_weight(c, c, k): the bilinear tent filter on the channel diagonal."""
    factor = (k + 1) // 2
    center = factor - 1 if k % 2 == 1 else factor - 0.5
    og = np.ogrid[:k, :k]
    filt = (1 - abs(og[0] - center) / factor) * (1 - abs(og[1] - center) / factor)
    w = np.zeros((c, c, k, k), dtype=np.float64)
    w[range(c), range(c), :, :] = filt
    return torch.from_numpy(w).float()


def fcn8_state_dict(num_classes, seed=0, dense_up=False):
    """Keys/shapes of models.FCN8(num_classes).state_dict(): 39 entries.  The upsamplers get the reference's bilinear
    weights, or (dense_up) random dense ones (a loaded state_dict may hold any weight)."""
    g = _Gen(seed, False)
    for _, stage, j, cin, cout in _features():
        if cout is not None:
            g.conv(f"{stage}.{j}", cout, cin, 3, bias=True)
    g.conv("adj_pool3", num_classes, 256, 1, bias=True)
    g.conv("adj_pool4", num_classes, 512, 1, bias=True)
    g.conv("output.0", 4096, 512, 7, bias=True)
    g.conv("output.3", 4096, 4096, 1, bias=True)
    g.conv("output.6", num_classes, 4096, 1, bias=True)
    for name, k in UPSAMPLERS:
        if dense_up:
            w = g.rs.standard_normal((num_classes, num_classes, k, k)).astype(np.float32) * np.float32(1.0 / num_classes)
            g.sd[name + ".weight"] = torch.from_numpy(w)
        else:
            g.sd[name + ".weight"] = upsampling_weight(num_classes, k)
    return g.sd


def fcn8_trunk(sd, x):
    """(pool3, pool4, pool5) of fcn.py:80-82."""
    taps = {}
    for fi, stage, j, _, cout in _features():
        if cout is None:
            x = F.max_pool2d(x, 2, 2, ceil_mode=True)
        else:
            x = F.relu(_conv(sd, f"{stage}.{j}", x, 1, 100 if fi == 0 else 1))
        taps[stage] = x
    return taps["pool3"], taps["pool4"], taps["pool5"]


def fcn8_forward(sd, x):
    """fcn.py:76-97.  Returns the fp32 logits [B, C, H, W] at the input resolution."""
    H, W = x.shape[2:]
    pool3, pool4, pool5 = fcn8_trunk(sd, x)
    out = F.relu(_conv(sd, "output.0", pool5))
    out = F.relu(_conv(sd, "output.3", out))
    out = _conv(sd, "output.6", out)
    up = F.conv_transpose2d(out, sd["up_output.weight"], stride=2)
    a4 = _conv(sd, "adj_pool4", 0.01 * pool4)
    s2 = F.conv_transpose2d(a4[:, :, 5:5 + up.shape[2], 5:5 + up.shape[3]] + up, sd["up_pool4_out.weight"], stride=2)
    a3 = _conv(sd, "adj_pool3", 0.0001 * pool3)
    f = F.conv_transpose2d(a3[:, :, 9:9 + s2.shape[2], 9:9 + s2.shape[3]] + s2, sd["up_final.weight"], stride=8)
    return f[:, :, 31:31 + H, 31:31 + W].contiguous()
