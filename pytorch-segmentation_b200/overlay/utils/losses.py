"""`utils.losses` overlay: the reference's loss registry (train.py:30 `getattr(losses, config['loss'])`) with
CrossEntropyLoss2d replaced by the sm_90a kernel version; the other losses are re-exported from the reference file."""
import importlib.util
import os

from . import REFERENCE_UTILS

if REFERENCE_UTILS is not None:
    _spec = importlib.util.spec_from_file_location("_reference_utils_losses", os.path.join(REFERENCE_UTILS, "losses.py"))
    _ref = importlib.util.module_from_spec(_spec)
    _spec.loader.exec_module(_ref)
    for _n in dir(_ref):
        if not _n.startswith("_"):
            globals()[_n] = getattr(_ref, _n)

from seg_b200.losses import CE_DiceLoss, CrossEntropyLoss2d, DiceLoss, LovaszSoftmax  # noqa: E402,F401
