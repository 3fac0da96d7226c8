"""Overlay for the reference's `models` registry (models/__init__.py): put this directory's PARENT
(`pytorch-segmentation_b200/overlay`) in front of the reference tree on PYTHONPATH and `train.py` resolves
`config['arch']['type']` == 'DeepLab' / 'PSPNet' to the H100-native classes while every other architecture keeps
coming from the reference, unmodified.  See INTEGRATION.md."""
import importlib
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(os.path.dirname(_HERE))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)


def _find_reference_models():
    root = os.environ.get("SEG_REFERENCE_ROOT")
    cands = [root] if root else []
    cands += [p or os.getcwd() for p in sys.path]
    for c in cands:
        d = os.path.join(c, "models")
        if os.path.isfile(os.path.join(d, "deeplabv3_plus.py")) and os.path.abspath(d) != _HERE:
            return d
    return None


_REF_MODELS = _find_reference_models()
if _REF_MODELS is not None:
    __path__.append(_REF_MODELS)  # submodules not overridden here (fcn, unet, segnet, ...) load from the reference
    for _mod, _names in (("fcn", ["FCN8"]), ("unet", ["UNet", "UNetResnet"]), ("segnet", ["SegNet", "SegResNet"]), ("enet", ["ENet"]),
                         ("gcn", ["GCN"]), ("duc_hdc", ["DeepLab_DUC_HDC"]), ("pspnet", ["PSPDenseNet"])):
        try:
            _m = importlib.import_module(f"{__name__}.{_mod}")
            for _n in _names:
                globals()[_n] = getattr(_m, _n)
        except Exception as _e:  # a reference model that cannot import here stays unavailable, as in the reference
            globals().setdefault("_import_errors", {})[_mod] = repr(_e)

from seg_b200.nets import DeepLab, PSPNet, UperNet  # noqa: E402,F401  H100-native replacements (same names, same contract)
