"""CPU oracle for the H100 segmentation hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional (state_dict-keyed) restatement, in plain PyTorch CPU ops, of the reference's hot path:
  models/deeplabv3_plus.py (ResNet trunk surgery :15-63, ASSP :253-297, Decoder :303-330, DeepLab.forward :356-362),
  torchvision.models.resnet Bottleneck (v1.5, stride on conv2), utils/losses.py, utils/lovasz_losses.py,
  utils/sync_batchnorm/batchnorm.py:128-145.
The arithmetic of the reference lives in third-party PyTorch/ATen (pinned torch==1.1.0, torchvision==0.3.0,
requirements.txt:1-2); this oracle calls the same ATen ops (F.conv2d, F.batch_norm, F.interpolate, ...) on CPU.

Pinning: the reference ships NO tests (SURVEY.md §4), so the oracle is pinned against outputs of the reference
itself: oracle/make_golden.py imports /root/reference unmodified, loads the oracle-generated state_dict with
strict=True (proves key names + shapes), runs forward/loss/backward and commits the results to tests/golden/*.npz;
tests/test_oracle_golden.py checks the oracle reproduces them.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this package.
"""
