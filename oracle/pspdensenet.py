"""PSPDenseNet (models/pspnet.py:117-205, trained from scratch) for the CPU oracle (TEST INFRASTRUCTURE — see
oracle/__init__.py): a deterministic state_dict factory with the reference's names and shapes, and a functional fp32
restatement of the forward pass.

  pspdensenet_forward -> pspnet.py:178-196: block0 = conv(3x3, s2, no padding) BN ReLU, then ONE conv(3x3, no padding) + BN
                         applied twice (block0.3 / block0.4 == block0.6 / block0.7), max-pool(3, 2, 1); torchvision
                         dense blocks (each layer: BN ReLU 1x1 BN ReLU 3x3 over the concat of everything before it in
                         the block); transition1 with AvgPool2d(2, 2), transition2 / 3 without; block3 / block4 conv2
                         dilated 2 / 4; no norm5; the PSP module (bins 1, 2, 3, 6) and the aux branch on transition3
The shared block0 BN updates its running statistics twice per training forward, as the reference's does.
"""
import torch
import torch.nn.functional as F

from .models import _bn, _conv
from .weights import _Gen

BLOCKS = {"densenet121": (6, 12, 24, 16), "densenet169": (6, 12, 32, 32), "densenet201": (6, 12, 48, 32)}
GROWTH, BN_SIZE = 32, 4
DILATION = (1, 1, 2, 4)


def widths(backbone):
    """(input, output) channels of each dense block."""
    out, c = [], 64
    for n in BLOCKS[backbone]:
        out.append((c, c + n * GROWTH))
        c = (c + n * GROWTH) // 2
    return out


def pspdensenet_state_dict(num_classes, backbone="densenet121", seed=0, randomize_bn=True, in_channels=3):
    """The reference's state_dict keys in order, block0.6 / block0.7 naming the same tensors as block0.3 / block0.4."""
    g = _Gen(seed, randomize_bn)
    g.conv("block0.0", 64, in_channels, 3)
    g.bn("block0.1", 64)
    g.conv("block0.3", 64, 64, 3)
    g.bn("block0.4", 64)
    for k in ("weight",):
        g.sd["block0.6." + k] = g.sd["block0.3." + k]
    for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
        g.sd["block0.7." + k] = g.sd["block0.4." + k]
    w = widths(backbone)
    for bi, n in enumerate(BLOCKS[backbone]):
        c0 = w[bi][0]
        for k in range(n):
            p = f"block{bi + 1}.denselayer{k + 1}."
            g.bn(p + "norm1", c0 + k * GROWTH)
            g.conv(p + "conv1", BN_SIZE * GROWTH, c0 + k * GROWTH, 1)
            g.bn(p + "norm2", BN_SIZE * GROWTH)
            g.conv(p + "conv2", GROWTH, BN_SIZE * GROWTH, 3)
    g.bn("transition1.norm", w[0][1])
    g.conv("transition1.conv", w[1][0], w[0][1], 1)
    for t in (2, 3):
        g.bn(f"transition{t}.0", w[t - 1][1])
        g.conv(f"transition{t}.2", w[t][0], w[t - 1][1], 1)
    m = w[3][1]
    for i in range(4):
        g.conv(f"master_branch.0.stages.{i}.1", m // 4, m, 1)
        g.bn(f"master_branch.0.stages.{i}.2", m // 4)
    g.conv("master_branch.0.bottleneck.0", m // 4, 2 * m, 3)
    g.bn("master_branch.0.bottleneck.1", m // 4)
    g.conv("master_branch.1", num_classes, m // 4, 1, bias=True)
    g.conv("auxiliary_branch.0", m // 4, w[3][0], 3)
    g.bn("auxiliary_branch.1", m // 4)
    g.conv("auxiliary_branch.4", num_classes, m // 4, 1, bias=True)
    return g.sd


def _dense_block(sd, bi, x, n, dil, train):
    feats = [x]
    for k in range(n):
        p = f"block{bi}.denselayer{k + 1}."
        h = F.relu(_bn(sd, p + "norm1", torch.cat(feats, 1), train))
        h = F.relu(_bn(sd, p + "norm2", _conv(sd, p + "conv1", h), train))
        feats.append(_conv(sd, p + "conv2", h, 1, dil, dil))
    return torch.cat(feats, 1)


def pspdensenet_forward(sd, x, backbone="densenet121", train=True, use_aux=True):
    """Training returns (out, aux); dropout is not modelled (the train parity runs it at p = 0)."""
    size = x.shape[2:]
    x = F.relu(_bn(sd, "block0.1", _conv(sd, "block0.0", x, 2), train))
    x = F.relu(_bn(sd, "block0.4", _conv(sd, "block0.3", x), train))
    x = F.relu(_bn(sd, "block0.7", _conv(sd, "block0.6", x), train))
    x = F.max_pool2d(x, 3, 2, 1)
    n = BLOCKS[backbone]
    x = _dense_block(sd, 1, x, n[0], DILATION[0], train)
    x = _conv(sd, "transition1.conv", F.relu(_bn(sd, "transition1.norm", x, train)))
    x = F.avg_pool2d(x, 2, 2)
    x = _dense_block(sd, 2, x, n[1], DILATION[1], train)
    x = _conv(sd, "transition2.2", F.relu(_bn(sd, "transition2.0", x, train)))
    x = _dense_block(sd, 3, x, n[2], DILATION[2], train)
    x_aux = _conv(sd, "transition3.2", F.relu(_bn(sd, "transition3.0", x, train)))
    x = _dense_block(sd, 4, x_aux, n[3], DILATION[3], train)
    h, w = x.shape[2:]
    pyr = [x]
    for i, bins in enumerate((1, 2, 3, 6)):
        p = F.adaptive_avg_pool2d(x, bins)
        p = F.relu(_bn(sd, f"master_branch.0.stages.{i}.2", _conv(sd, f"master_branch.0.stages.{i}.1", p), train))
        pyr.append(F.interpolate(p, size=(h, w), mode="bilinear", align_corners=True))
    y = _conv(sd, "master_branch.0.bottleneck.0", torch.cat(pyr, 1), 1, 1)
    y = F.relu(_bn(sd, "master_branch.0.bottleneck.1", y, train))
    out = F.interpolate(_conv(sd, "master_branch.1", y), size=size, mode="bilinear", align_corners=False)
    if train and use_aux:
        a = F.relu(_bn(sd, "auxiliary_branch.1", _conv(sd, "auxiliary_branch.0", x_aux, 1, 1), train))
        aux = F.interpolate(_conv(sd, "auxiliary_branch.4", a), size=size, mode="bilinear", align_corners=False)
        return out, aux
    return out
