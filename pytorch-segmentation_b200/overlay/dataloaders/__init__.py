"""Overlay for the reference's `dataloaders` registry (train.py:21-22 `getattr(dataloaders, config[...]['type'])`):
`CityScapes`, `VOC` and `ADE20K` are the reference's loaders over datasets in device mode — the worker decodes the
sample to uint8, makes the reference's random draws and packs the batch (seg_b200.data.device_collate); the device
prefetcher (the `base` overlay's DataPrefetcher) copies it once and runs one augmentation kernel.  `COCO` and
`DeepScene` are the reference's, unchanged.  See INTEGRATION.md."""
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(os.path.dirname(_HERE))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)


def _find_reference_dataloaders():
    root = os.environ.get("SEG_REFERENCE_ROOT")
    cands = [root] if root else []
    cands += [p or os.getcwd() for p in sys.path]
    for c in cands:
        d = os.path.join(c, "dataloaders")
        if os.path.isfile(os.path.join(d, "cityscapes.py")) and os.path.abspath(d) != _HERE:
            return d
    return None


REFERENCE_DATALOADERS = _find_reference_dataloaders()
if REFERENCE_DATALOADERS is not None:
    __path__.append(REFERENCE_DATALOADERS)  # coco, deepscene and the label files load from the reference
    from .coco import COCO  # noqa: E402,F401
    from .deepscene import DeepScene  # noqa: E402,F401
    from ._device import ADE20K, VOC, CityScapes  # noqa: E402,F401
