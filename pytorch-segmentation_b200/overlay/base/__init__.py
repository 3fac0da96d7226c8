"""Overlay for the reference's `base` package: BaseModel, BaseTrainer, BaseDataSet, BaseDataLoader and every other name
are the reference's own objects; `DataPrefetcher` (trainer.py:7,30-33) is the device prefetcher, which runs the packed
batches of the `dataloaders` overlay through the sm_90a augmentation kernels and passes float batches through unchanged.
See INTEGRATION.md."""
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(os.path.dirname(_HERE))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)


def _find_reference_base():
    root = os.environ.get("SEG_REFERENCE_ROOT")
    cands = [root] if root else []
    cands += [p or os.getcwd() for p in sys.path]
    for c in cands:
        d = os.path.join(c, "base")
        if os.path.isfile(os.path.join(d, "base_dataset.py")) and os.path.abspath(d) != _HERE:
            return d
    return None


REFERENCE_BASE = _find_reference_base()
if REFERENCE_BASE is not None:
    __path__.append(REFERENCE_BASE)
    # the reference's names first: seg_b200.nets imports BaseModel from this package
    from .base_dataloader import *  # noqa: E402,F401,F403
    from .base_dataset import *  # noqa: E402,F401,F403
    from .base_model import *  # noqa: E402,F401,F403
    from .base_trainer import *  # noqa: E402,F401,F403

from seg_b200.data import DevicePrefetcher as DataPrefetcher  # noqa: E402,F401
