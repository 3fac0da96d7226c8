"""seg_b200 — H100-native forward/backward engine for the data-parallel hot path of yassouali/pytorch-segmentation.

Host side mirrors the reference's plugin surface (models / losses registries); all arithmetic runs in the hand-written
sm_90a kernels of ``libseg_b200.so`` (C ABI: include/seg_b200.h).  No CPU fallback.

Attributes are resolved lazily so that ``python -m seg_b200.launch`` can order sys.path (overlay before the reference
tree) before anything imports the reference's ``base`` / ``utils`` packages.
"""
_LAZY = {
    "DeepLab": ("nets", "DeepLab"),
    "PSPNet": ("nets", "PSPNet"),
    "UperNet": ("nets", "UperNet"),
    "CrossEntropyLoss2d": ("losses", "CrossEntropyLoss2d"),
    "DiceLoss": ("losses", "DiceLoss"),
    "CE_DiceLoss": ("losses", "CE_DiceLoss"),
    "LovaszSoftmax": ("losses", "LovaszSoftmax"),
    "eval_metrics": ("metrics", "eval_metrics"),
    "AverageMeter": ("metrics", "AverageMeter"),
    "FusedTrainStep": ("train", "FusedTrainStep"),
}

__all__ = list(_LAZY) + ["lib", "ops", "nets", "losses", "engine", "comm", "train", "launch", "lr_scheduler", "data", "inference"]


def __getattr__(name):
    import importlib
    if name in _LAZY:
        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(f"{__name__}.{mod}"), attr)
    if name in ("lib", "ops", "nets", "losses", "engine", "comm", "train", "launch", "lr_scheduler", "data", "inference"):
        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
