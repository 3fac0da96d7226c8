"""The drop-in overlay: with `seg_b200.launch` ordering sys.path as [overlay, reference root], the
reference's own registries resolve DeepLab / PSPNet / CrossEntropyLoss2d to the H100-native classes and everything else
to the reference's.  Runs against the unmodified reference tree that build() packs into oracle/_ref/reference.zip
(oracle/install_ref.sh), extracted to a temporary directory; skipped where build() had no reference checkout to pack."""
import os
import subprocess
import sys
import zipfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_ZIP = os.path.join(ROOT, "oracle", "_ref", "reference.zip")

CODE = r"""
import sys
from seg_b200 import launch
launch.setup_paths(sys.argv[1])
import models, seg_b200
from utils import losses, lr_scheduler, helpers, metrics
assert metrics.eval_metrics is seg_b200.eval_metrics and metrics.AverageMeter is seg_b200.AverageMeter
assert hasattr(metrics, 'batch_pix_accuracy') and losses.LovaszSoftmax is seg_b200.LovaszSoftmax
assert models.DeepLab is seg_b200.DeepLab and models.PSPNet is seg_b200.PSPNet, (models.DeepLab, models.PSPNet)
assert models.UNet.__module__.endswith('unet') and 'reference' in models.UNet.__init__.__code__.co_filename
assert losses.CrossEntropyLoss2d is seg_b200.CrossEntropyLoss2d
assert hasattr(losses, 'DiceLoss') and hasattr(losses, 'LovaszSoftmax') and hasattr(lr_scheduler, 'Poly')
from base import BaseModel
m = models.DeepLab(19, backbone='resnet50', pretrained=False, freeze_bn=False, freeze_backbone=False, output_stride=16)
assert isinstance(m, BaseModel)
# exactly what train.py:14-16,26,30 and base_trainer.py:46-57 do
import json
import os
cfg = json.load(open(os.path.join(sys.argv[1], 'config.json')))
cfg['arch']['args']['pretrained'] = False
cfg['arch']['type'], cfg['arch']['args']['backbone'] = 'PSPNet', 'resnet50'
model = getattr(models, cfg['arch']['type'])(21, **cfg['arch']['args'])
loss = getattr(losses, cfg['loss'])(ignore_index=cfg['ignore_index'])
groups = [{'params': model.get_decoder_params()}, {'params': model.get_backbone_params(), 'lr': 0.001}]
import torch
opt = torch.optim.SGD(groups, lr=0.01, momentum=0.9, weight_decay=1e-4)
assert sum(len(g['params']) for g in opt.param_groups) == len(list(model.parameters()))
# base/base_trainer.py:11-12,33-35: config['use_synch_bn'] -> convert_model + DataParallelWithCallback from utils.sync_batchnorm
from utils.sync_batchnorm import convert_model, DataParallelWithCallback, SynchronizedBatchNorm2d
assert model.use_sync_bn is False and convert_model(model) is model and model.use_sync_bn is True   # engine model: marked, BN holders kept
assert all(not isinstance(mm, SynchronizedBatchNorm2d) for mm in model.modules())
import torch.nn as nn
plain = convert_model(nn.Sequential(nn.Conv2d(3, 4, 1), nn.BatchNorm2d(4)))                         # anything else: the reference's conversion
assert isinstance(plain[1], SynchronizedBatchNorm2d)
assert issubclass(DataParallelWithCallback, nn.DataParallel)
print(str(model).splitlines()[-1])
print('OVERLAY_OK')
"""


@pytest.mark.skipif(not os.path.isfile(REF_ZIP), reason="oracle/_ref/reference.zip not built (build() found no reference checkout)")
def test_overlay_resolves_registries(tmp_path):
    ref = tmp_path / "reference"
    with zipfile.ZipFile(REF_ZIP) as z:
        z.extractall(ref)
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "pytorch-segmentation_b200")
    r = subprocess.run([sys.executable, "-W", "ignore", "-c", CODE, str(ref)], env=env, cwd=str(ref), capture_output=True, text=True,
                       timeout=600)
    assert "OVERLAY_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    assert "Nbr of trainable parameters: 51446762" in r.stdout


def test_constructor_defaults_match_the_reference():
    """A config that omits `backbone` must build the architecture the reference would (models/deeplabv3_plus.py:337,
    models/pspnet.py:42, models/upernet.py:121); `pretrained` cannot be honoured offline: the default only warns."""
    import inspect
    import logging
    import seg_b200
    want = {"DeepLab": "xception", "PSPNet": "resnet152", "UperNet": "resnet101"}
    for name, backbone in want.items():
        sig = inspect.signature(getattr(seg_b200, name).__init__)
        assert sig.parameters["backbone"].default == backbone, name
        assert sig.parameters["pretrained"].default is None, name
        assert list(sig.parameters)[1:3] == ["num_classes", "in_channels"], name
    records = []
    h = logging.Handler()
    h.emit = records.append
    logging.getLogger("DeepLab").addHandler(h)
    try:
        seg_b200.DeepLab(5, backbone="resnet50")                    # default pretrained -> warning, random init
        n = len(records)
        seg_b200.DeepLab(5, backbone="resnet50", pretrained=False)  # explicit False -> silent
    finally:
        logging.getLogger("DeepLab").removeHandler(h)
    assert n >= 1 and len(records) == n and "ImageNet" in records[0].getMessage()
    with pytest.raises(RuntimeError, match="network"):
        seg_b200.DeepLab(5, backbone="resnet50", pretrained=True)
