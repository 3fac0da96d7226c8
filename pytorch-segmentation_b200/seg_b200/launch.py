"""Run an UNMODIFIED reference script (train.py / inference.py) with the H100-native models and losses plugged in:

    cd /path/to/pytorch-segmentation
    PYTHONPATH=/path/to/repo/pytorch-segmentation_b200 python -m seg_b200.launch train.py -c config.json

`python train.py` puts the script's own directory first on sys.path, ahead of PYTHONPATH, so the overlay packages
(`overlay/models`, `overlay/utils`) could never win there; this launcher orders sys.path as
[overlay, reference root, ...] and then executes the script as __main__ — the script's source is untouched.
Under torchrun (one process per GPU; `torchrun --nproc-per-node N -m seg_b200.launch train.py -c config.json` with
`n_gpu: 1` in the config) every process becomes a data-parallel replica: its own GPU is device 0, the NCCL process group
is up, gradients are all-reduced inside `loss.backward()`, the loss is the global-batch mean and `use_synch_bn` turns on
the NVLink statistics exchange (`init_data_parallel`).
"""
import os
import runpy
import sys


def setup_paths(reference_root):
    here = os.path.dirname(os.path.abspath(__file__))
    pkg = os.path.dirname(here)
    overlay = os.path.join(pkg, "overlay")
    reference_root = os.path.abspath(reference_root)
    os.environ.setdefault("SEG_REFERENCE_ROOT", reference_root)
    for p in (reference_root, pkg, overlay):  # final order: overlay, pkg, reference root
        while p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    # anything of the reference imported before the path was ordered must be re-resolved through the overlay
    for name in list(sys.modules):
        if name.split(".")[0] in ("models", "utils", "base", "dataloaders"):
            del sys.modules[name]
    # utils/transforms.py:4 imports skimage, which this image lacks; the trainer never calls it (SURVEY.md §8c shim 1)
    try:
        import skimage  # noqa: F401
    except Exception:
        import types
        for n in ("skimage", "skimage.filters"):
            sys.modules.setdefault(n, types.ModuleType(n))
        sys.modules["skimage.filters"].gaussian = None


def init_data_parallel():
    """Under torchrun (one process per GPU) make this process a data-parallel replica of an UNMODIFIED train.py.

    * The reference hard-codes `cuda:0` and `device_ids = range(n_gpu)` (base/base_trainer.py:176-187), so every process
      must see ITS GPU as device 0 — but all GPUs have to stay visible for the NVLink peer-memory exchange (CUDA IPC) and
      NCCL: CUDA_VISIBLE_DEVICES is rotated ([local, local+1, ..., local-1]) rather than restricted.  Run the config with
      `n_gpu: 1`: its DataParallel-of-one wrapper (base/base_trainer.py:33-38) is then a pass-through.
    * The NCCL process group is initialised here; from then on the engine's autograd nodes all-reduce (mean) the flat
      gradient buffer inside `loss.backward()`, `CrossEntropyLoss2d` reports the global-batch mean, and — when the config
      says `use_synch_bn` — the overlay's `convert_model` makes the engine exchange BatchNorm statistics over NVLink
      (seg_b200/nets.py `_EngineFn`, seg_b200/losses.py `_CEFn`, overlay/utils/sync_batchnorm.py).  Identical replicas in,
      identical replicas out: what nn.DataParallel guarantees in the reference.
    Returns (rank, world)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 or "LOCAL_RANK" not in os.environ:
        return 0, 1
    local = int(os.environ["LOCAL_RANK"])
    if "CUDA_VISIBLE_DEVICES" in os.environ:
        devs = [d for d in os.environ["CUDA_VISIBLE_DEVICES"].split(",") if d != ""]
    else:
        n = int(os.environ.get("LOCAL_WORLD_SIZE", world))
        devs = [str(i) for i in range(n)]
    if os.environ.get("SEG_DEVICES_ROTATED") != "1" and len(devs) > 1:
        k = local % len(devs)
        os.environ["CUDA_VISIBLE_DEVICES"] = ",".join(devs[k:] + devs[:k])
        os.environ["SEG_DEVICES_ROTATED"] = "1"
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", 0))
    return dist.get_rank(), dist.get_world_size()


def main():
    if len(sys.argv) < 2:
        print(__doc__)
        sys.exit(2)
    script = os.path.abspath(sys.argv[1])
    setup_paths(os.path.dirname(script))
    init_data_parallel()
    if os.environ.get("SEG_FUSED_OPTIM", "1") != "0":
        # base/base_trainer.py:57 builds getattr(torch.optim, config['optimizer']['type']): "SGD" over CUDA fp32
        # parameters resolves to the torch.optim.SGD subclass whose step() is the multi-tensor kernel (same param_groups /
        # state_dict / schedulers); any other use gets the stock class
        from seg_b200 import optim
        optim.install()
    sys.argv = [script] + sys.argv[2:]
    try:
        runpy.run_path(script, run_name="__main__")
    finally:
        _teardown_data_parallel()


def _teardown_data_parallel(grace_s=20.0):
    """After the script: captured graphs hold this process group's NCCL kernels, and a communicator torn down (explicitly or
    by the interpreter's exit handlers) while one is alive blocks forever (measured in tests/dp_worker.py).  Release every
    engine graph first; if the teardown still does not return within `grace_s`, flush logging and leave hard."""
    if "torch.distributed" not in sys.modules:
        return
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() <= 1:
        return
    import logging
    import threading
    from seg_b200.nets import release_all_graphs
    release_all_graphs()

    def _bail():
        logging.shutdown()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(0)
    t = threading.Timer(grace_s, _bail)
    t.daemon = True
    t.start()
    dist.destroy_process_group()
    t.cancel()


if __name__ == "__main__":
    main()
