"""`utils.sync_batchnorm` overlay (imported by base/base_trainer.py:11-12): the reference's package, re-exported, with
`convert_model` made aware of the H100-native engine models.

The reference turns `config['use_synch_bn']` into `convert_model(model)` + `DataParallelWithCallback(model, device_ids)`
(base/base_trainer.py:33-35): every nn.BatchNorm2d is swapped for a SynchronizedBatchNorm2d whose replicas meet through
Python queues (sync_batchnorm/batchnorm.py:105-126).  An engine model's BatchNorm modules are parameter HOLDERS — its
statistics come out of the conv epilogues — so there is nothing to swap: `convert_model` marks the model instead
(`use_sync_bn = True`) and the engine exchanges the per-channel sums between the one-process-per-GPU replicas with its
one-shot NVLink peer-memory kernel (`seg_syncbn_exchange`), reproducing the reference's clamp(var, eps) formula
(batchnorm.py:145).  Any other model goes through the reference's own convert_model, unchanged.
"""
import importlib.util
import os
import sys

from . import REFERENCE_UTILS

_ref = None
if REFERENCE_UTILS is not None:
    _dir = os.path.join(REFERENCE_UTILS, "sync_batchnorm")
    _spec = importlib.util.spec_from_file_location("_reference_sync_batchnorm", os.path.join(_dir, "__init__.py"),
                                                   submodule_search_locations=[_dir])
    _ref = importlib.util.module_from_spec(_spec)
    sys.modules["_reference_sync_batchnorm"] = _ref
    _spec.loader.exec_module(_ref)
    for _n in dir(_ref):
        if not _n.startswith("_"):
            globals()[_n] = getattr(_ref, _n)


def _engine_models(module):
    from seg_b200.nets import _EngineModel
    return [m for m in module.modules() if isinstance(m, _EngineModel)]


def convert_model(module):
    engines = _engine_models(module)
    if engines:
        for m in engines:
            m.use_sync_bn = True
        return module
    if _ref is None:
        raise RuntimeError("utils.sync_batchnorm overlay: reference tree not found (set SEG_REFERENCE_ROOT)")
    return _ref.convert_model(module)
