"""Overlay for the reference's `utils` package: everything resolves to the reference's modules except `utils.losses`,
whose CrossEntropyLoss2d is the H100-native one.  See INTEGRATION.md."""
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(os.path.dirname(_HERE))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)


def _find_reference_utils():
    root = os.environ.get("SEG_REFERENCE_ROOT")
    cands = [root] if root else []
    cands += [p or os.getcwd() for p in sys.path]
    for c in cands:
        d = os.path.join(c, "utils")
        if os.path.isfile(os.path.join(d, "lovasz_losses.py")) and os.path.abspath(d) != _HERE:
            return d
    return None


REFERENCE_UTILS = _find_reference_utils()
if REFERENCE_UTILS is not None:
    __path__.append(REFERENCE_UTILS)
    from .logger import Logger  # noqa: E402,F401  the reference package's own export (train.py:9 `from utils import Logger`)
