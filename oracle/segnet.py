"""SegNet (models/segnet.py:13-132) for the CPU oracle (TEST INFRASTRUCTURE — see oracle/__init__.py): a deterministic
state_dict factory with the reference's names and shapes, and a functional fp32 restatement of the forward pass.

  segnet_forward -> segnet.py:84-120 (SegNet.forward): the VGG16-BN encoder (vgg16_bn's features without the pools), five
                    MaxPool2d(2, 2, return_indices=True) and five MaxUnpool2d(2, 2) to the encoder maps' sizes
"""
import torch.nn.functional as F

from .models import _bn, _conv
from .weights import _Gen

# output channels of the (conv 3x3 p1 + bias, BN, ReLU) triples of each stage, and each stage's input channels
ENCODER = ((64, 64), (128, 128), (256, 256, 256), (512, 512, 512), (512, 512, 512))
DECODER_IN = (512, 512, 256, 128, 64)
DECODER = ((512, 512, 512), (512, 512, 256), (256, 256, 128), (128, 64), (64, 64))


def _stages(in_channels):
    """[(stage name, [(module index, cin, cout)])] in the reference's registration order."""
    out, cin = [], in_channels
    for i, widths in enumerate(ENCODER):
        out.append((f"stage{i + 1}_encoder", [(3 * j, c0, c1) for j, (c0, c1) in enumerate(zip((cin,) + widths[:-1], widths))]))
        cin = widths[-1]
    for i, (c, widths) in enumerate(zip(DECODER_IN, DECODER)):
        out.append((f"stage{i + 1}_decoder", [(3 * j, c0, c1) for j, (c0, c1) in enumerate(zip((c,) + widths[:-1], widths))]))
    return out


def segnet_state_dict(num_classes, in_channels=3, seed=0, randomize_bn=False):
    """Keys/shapes of models.SegNet(num_classes, in_channels).state_dict(): 184 entries, 106 parameters."""
    g = _Gen(seed, randomize_bn)
    for stage, convs in _stages(in_channels):
        for j, cin, cout in convs:
            g.conv(f"{stage}.{j}", cout, cin, 3, bias=True)
            g.bn(f"{stage}.{j + 1}", cout)
    g.conv("stage5_decoder.6", num_classes, 64, 3, bias=True)
    return g.sd


def _stage(sd, stage, convs, x, train):
    for j, _, _ in convs:
        x = F.relu(_bn(sd, f"{stage}.{j + 1}", _conv(sd, f"{stage}.{j}", x, 1, 1), train))
    return x


def segnet_forward(sd, x, train=True):
    """segnet.py:84-120.  Returns the fp32 logits [B, C, H, W] at the input resolution."""
    stages = _stages(sd["stage1_encoder.0.weight"].shape[1])
    saved = []
    for stage, convs in stages[:5]:
        x = _stage(sd, stage, convs, x, train)
        size = x.shape[2:]
        x, idx = F.max_pool2d(x, 2, 2, return_indices=True)
        saved.append((idx, size))
    for (stage, convs), (idx, size) in zip(stages[5:], reversed(saved)):
        x = _stage(sd, stage, convs, F.max_unpool2d(x, idx, 2, 2, output_size=size), train)
    return _conv(sd, "stage5_decoder.6", x, 1, 1)
