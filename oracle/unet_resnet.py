"""UNetResnet (models/unet.py:126-209) for the CPU oracle (TEST INFRASTRUCTURE — see oracle/__init__.py): a deterministic
state_dict factory with the reference's names and shapes, and a functional fp32 restatement of the forward pass, in the style
of oracle/weights.py and oracle/models.py.

  unet_resnet_forward -> unet.py:172-204 (UNetResnet.forward) over the deep-stem dilated ResNet of resnet.py:136-163,190-210
                         (the trunk of oracle.models.pspnet_forward)
"""
import torch
import torch.nn.functional as F

from .models import _bn, _bottleneck, _conv
from .weights import RESNET_LAYERS, _Gen, pspnet_state_dict

# unet.py:146-164: (name, in channels, out channels); upconvN are ConvTranspose2d(4, 2, 1, bias=False), the rest 3x3 convs
# with bias
DECODER = (("conv1", 2048, 192), ("upconv1", 192, 128), ("conv2", 1152, 128), ("upconv2", 128, 96), ("conv3", 608, 96),
           ("upconv3", 96, 64), ("conv4", 320, 64), ("upconv4", 64, 48), ("conv5", 48, 48), ("upconv5", 48, 32),
           ("conv6", 32, 32))
TRUNK_PLAN = {1: (1, 1, 1), 2: (2, 1, 1), 3: (1, 1, 2), 4: (1, 2, 4)}  # (first-block stride, first-block dil, other dil)


def unet_resnet_state_dict(num_classes, backbone="resnet50", seed=0, randomize_bn=False):
    """Keys/shapes of models.UNetResnet(num_classes, backbone=backbone, pretrained=False).state_dict(): 348 entries for
    resnet50.  The trunk is PSPNet's (same seed, same values); the decoder's weights come from a second generator."""
    sd = {k: v for k, v in pspnet_state_dict(num_classes, backbone, seed, randomize_bn, use_aux=False).items()
          if k.startswith(("initial.", "layer"))}
    g = _Gen(seed + 7919, randomize_bn)
    for name, cin, cout in DECODER:
        if name.startswith("up"):
            g.conv(name, cin, cout, 4)  # ConvTranspose2d weight [in, out, k, k]
        else:
            g.conv(name, cout, cin, 3, bias=True)
    g.conv("conv7", num_classes, 32, 1)
    sd.update(g.sd)
    return sd


def _resample(x, size):
    """F.interpolate(bilinear, align_corners=True) to `size` (unet.py:178,183,187,195-196)."""
    return F.interpolate(x, size=tuple(size), mode="bilinear", align_corners=True)


def _up(sd, name, x):
    return F.conv_transpose2d(x, sd[name + ".weight"], None, 2, 1)


def unet_resnet_forward(sd, x, backbone="resnet50", train=True):
    """unet.py:172-204.  Returns the fp32 logits [B, C, H, W] at the input resolution."""
    H, W = x.shape[2:]
    y = F.relu(_bn(sd, "initial.0.1", _conv(sd, "initial.0.0", x, 2, 1), train))
    y = F.relu(_bn(sd, "initial.0.4", _conv(sd, "initial.0.3", y, 1, 1), train))
    y = F.relu(_bn(sd, "initial.1", _conv(sd, "initial.0.6", y, 1, 1), train))
    y = F.max_pool2d(y, 3, 2, 1)
    feats = []
    for li in (1, 2, 3, 4):
        stride, d0, d = TRUNK_PLAN[li]
        for b in range(RESNET_LAYERS[backbone][li - 1]):
            y = _bottleneck(sd, f"layer{li}.{b}.", y, stride if b == 0 else 1, d0 if b == 0 else d, train)
        feats.append(y)
    x1, x2, x3, x4 = feats
    y = _up(sd, "upconv1", _conv(sd, "conv1", x4, 1, 1))
    y = torch.cat([_resample(y, x3.shape[2:]), x3], 1)
    y = _up(sd, "upconv2", _conv(sd, "conv2", y, 1, 1))
    y = torch.cat([_resample(y, x2.shape[2:]), x2], 1)
    y = _up(sd, "upconv3", _conv(sd, "conv3", y, 1, 1))
    y = torch.cat([_resample(y, x1.shape[2:]), x1], 1)
    y = _up(sd, "upconv4", _conv(sd, "conv4", y, 1, 1))
    y = _up(sd, "upconv5", _conv(sd, "conv5", y, 1, 1))
    if y.shape[2:] != (H, W):
        y = _resample(y, (H, W))
    return _conv(sd, "conv7", _conv(sd, "conv6", y, 1, 1))
