"""DeepLab_DUC_HDC (models/duc_hdc.py) for the CPU oracle (TEST INFRASTRUCTURE — see oracle/__init__.py): a deterministic
state_dict factory with the reference's names and shapes, and a functional fp32 restatement of the forward pass, in the style
of oracle/weights.py and oracle/models.py.

  duc_hdc_forward -> duc_hdc.py:228-234 (DeepLab_DUC_HDC.forward), :105-113 (ResNet_HDC_DUC.forward with the HDC surgery of
                     :76-103), :157-174 (ASSP.forward), :200-208 (Decoder.forward), :28-31 (DUC.forward)
"""
import numpy as np
import torch
import torch.nn.functional as F

from .models import _bn, _bottleneck, _conv
from .weights import RESNET_LAYERS, _Gen, _tv_bottleneck_layers

ASPP_DILATIONS = (1, 6, 12, 18, 24, 36)  # duc_hdc.py:132
HDC_DILATIONS = {1: [1] * 3, 2: [1] * 4, 3: [1, 2, 3] * 7 + [2, 2], 4: [3, 4, 5]}  # duc_hdc.py:84-85 (layers 1, 2: torchvision's)
LAYER_STRIDES = {1: 1, 2: 2, 3: 1, 4: 1}  # duc_hdc.py:88-103 set layer3 / layer4 to stride 1


def duc_hdc_state_dict(num_classes, seed=0, randomize_bn=False, in_channels=3, icnr=True):
    """Keys/shapes of models.DeepLab_DUC_HDC(num_classes, pretrained=False).state_dict() (duc_hdc.py:214-224): 704 entries.
    icnr: DUC_out.conv gets the ICNR pattern of duc_hdc.py:33-49 (the r*r channels of a shuffle group share one kernel)."""
    g = _Gen(seed, randomize_bn)
    g.conv("backbone.layer0.0", 64, in_channels, 7)
    g.bn("backbone.layer0.1", 64)
    _tv_bottleneck_layers(g, "backbone.", RESNET_LAYERS["resnet101"])
    for i, d in enumerate(ASPP_DILATIONS, 1):
        g.conv(f"ASSP.aspp{i}.0", 256, 2048, 1 if i == 1 else 3)
        g.bn(f"ASSP.aspp{i}.1", 256)
    g.conv("ASSP.avg_pool.1", 256, 2048, 1)
    g.bn("ASSP.avg_pool.2", 256)
    g.conv("ASSP.conv1", 256, 256 * 7, 1)
    g.bn("ASSP.bn1", 256)
    g.conv("decoder.conv1", 48, 256, 1)
    g.bn("decoder.bn1", 48)
    g.conv("decoder.DUC.conv", 256 * 4, 256, 1)
    g.bn("decoder.DUC.bn", 256 * 4)
    g.conv("decoder.output.0", 256, 304, 3)
    g.bn("decoder.output.1", 256)
    g.conv("decoder.output.3", 256, 256, 3)
    g.bn("decoder.output.4", 256)
    g.conv("decoder.output.7", num_classes, 256, 1, bias=True)
    g.conv("DUC_out.conv", num_classes * 16, num_classes, 1)
    if icnr:
        w = g.sd["DUC_out.conv.weight"]
        g.sd["DUC_out.conv.weight"] = w[::16].repeat_interleave(16, dim=0).contiguous()
    g.bn("DUC_out.bn", num_classes * 16)
    return g.sd


def _duc(sd, name, x, r, train):
    """DUC.forward (duc_hdc.py:28-31): 1x1 conv (no bias) -> BN -> ReLU -> PixelShuffle(r)."""
    return F.pixel_shuffle(F.relu(_bn(sd, name + ".bn", _conv(sd, name + ".conv", x), train)), r)


def duc_hdc_forward(sd, x, output_stride=8, train=True, dropout=False):
    """duc_hdc.py:228-234.  Returns the fp32 output [B, C, 4*Hl, 4*Wl] (Hl, Wl: the layer1 size), ReLU'd as in the reference."""
    x = _conv(sd, "backbone.layer0.0", x, 2 if output_stride == 8 else 1, 3)
    x = F.relu(_bn(sd, "backbone.layer0.1", x, train))
    x = F.max_pool2d(x, 3, 2, 1)
    low = None
    for li in (1, 2, 3, 4):
        for b, d in enumerate(HDC_DILATIONS[li]):
            x = _bottleneck(sd, f"backbone.layer{li}.{b}.", x, LAYER_STRIDES[li] if b == 0 else 1, d, train)
        if li == 1:
            low = x
    outs = []
    for i, d in enumerate(ASPP_DILATIONS, 1):
        y = _conv(sd, f"ASSP.aspp{i}.0", x, 1, 0 if i == 1 else d, d)
        outs.append(F.relu(_bn(sd, f"ASSP.aspp{i}.1", y, train)))
    p = F.adaptive_avg_pool2d(x, 1)
    p = F.relu(_bn(sd, "ASSP.avg_pool.2", _conv(sd, "ASSP.avg_pool.1", p), train))
    outs.append(F.interpolate(p, size=x.shape[2:], mode="bilinear", align_corners=True))
    y = F.relu(_bn(sd, "ASSP.bn1", _conv(sd, "ASSP.conv1", torch.cat(outs, 1)), train))
    if dropout and train:
        y = F.dropout(y, 0.5, True)
    low = F.relu(_bn(sd, "decoder.bn1", _conv(sd, "decoder.conv1", low), train))
    u = _duc(sd, "decoder.DUC", y, 2, train)[:, :, : low.shape[2], : low.shape[3]]  # duc_hdc.py:204-206: always cropped
    y = torch.cat((low, u), 1)
    y = F.relu(_bn(sd, "decoder.output.1", _conv(sd, "decoder.output.0", y, 1, 1), train))
    y = F.relu(_bn(sd, "decoder.output.4", _conv(sd, "decoder.output.3", y, 1, 1), train))
    if dropout and train:
        y = F.dropout(y, 0.1, True)
    y = _conv(sd, "decoder.output.7", y)
    return _duc(sd, "DUC_out", y, 4, train)


def is_icnr(w, r):
    """True when the r*r output channels of every shuffle group of a [o, i, 1, 1] conv weight share one kernel."""
    o = w.shape[0]
    v = np.asarray(w.detach().reshape(o // (r * r), r * r, -1))
    return bool((v == v[:, :1]).all())
