"""H100-native drop-in models for the reference's plugin surface (models/__init__.py registry):

    DeepLab(num_classes, in_channels=3, backbone='xception',  pretrained=None, output_stride=16, freeze_bn=False, **_)
    PSPNet (num_classes, in_channels=3, backbone='resnet152', pretrained=None, use_aux=True,   freeze_bn=False, **_)
    UperNet(num_classes, in_channels=3, backbone='resnet101', pretrained=None, use_aux=True, fpn_out=256, freeze_bn=False, **_)
    DeepLab_DUC_HDC(num_classes, in_channels=3, pretrained=None, output_stride=8, freeze_bn=False, **_)
    UNetResnet(num_classes, in_channels=3, backbone='resnet50', pretrained=None, freeze_bn=False, **_)
    SegNet(num_classes, in_channels=3, pretrained=None, freeze_bn=False, freeze_backbone=False, **_)
    FCN8(num_classes, pretrained=None, freeze_bn=False, freeze_backbone=False, **_)
    PSPDenseNet(num_classes, in_channels=3, backbone='densenet201', pretrained=None, use_aux=True, freeze_bn=False, **_)

(default backbones are the reference's; `pretrained`: the reference defaults to True and downloads ImageNet weights — there is
no network here, so an explicit True raises and the default (None) initialises randomly with a logged warning)

Same constructor contract, same `state_dict()` keys and OIHW fp32 parameter layout, same `get_backbone_params /
get_decoder_params / freeze_bn` methods and the same forward contract (fp32 NCHW logits at input resolution; PSPNet
returns `(out, aux)` in training; DeepLab_DUC_HDC's are at 4x its layer1 size) as models/deeplabv3_plus.py:336-377 and
models/pspnet.py:41-105 — so train.py,
BaseTrainer (base/base_trainer.py:46-57), torch.optim.SGD, checkpoints and `convert_model` keep working.

The nn.Conv2d / nn.BatchNorm2d children are PARAMETER HOLDERS only: forward never calls them.  `forward` runs the
hand-written sm_90a kernels through `engine.Tape`; gradients reach the parameters through one autograd.Function.
There is no CPU / eager path: a CPU input raises.
"""
import logging
import math
import weakref
from itertools import chain

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .engine import Act, BilinearHead, ConvSpec, DwSpec, FullResHead, ShuffleHead, Tape
from .lib import IMPL_AUTO, require_device

try:  # inside the reference tree: subclass its BaseModel so isinstance checks and logging behave identically
    from base import BaseModel as _RefBaseModel  # type: ignore
except Exception:  # standalone (tests, bench, GPU box): API-compatible stand-in for base/base_model.py:6-23
    _RefBaseModel = None


_LIVE_MODELS = weakref.WeakSet()  # every engine model alive in this process (release_all_graphs)


def release_all_graphs():
    """Drop every captured CUDA graph of every live engine model.  Needed before an NCCL process group is torn down: a graph
    that captured the gradient all-reduce keeps the communicator's kernels alive and ncclCommDestroy blocks on it
    (seg_b200.launch calls this after the reference script returns)."""
    import gc
    for m in list(_LIVE_MODELS):
        if hasattr(m, "release_graphs"):
            m.release_graphs()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()


class BaseModel(nn.Module if _RefBaseModel is None else _RefBaseModel):
    def __init__(self):
        super().__init__()
        _LIVE_MODELS.add(self)
        if not hasattr(self, "logger"):
            self.logger = logging.getLogger(self.__class__.__name__)

    def _n_trainable(self):
        return int(sum(np.prod(p.size()) for p in self.parameters() if p.requires_grad))

    def summary(self):
        self.logger.info(f"Nbr of trainable parameters: {self._n_trainable()}")

    def __str__(self):
        return nn.Module.__str__(self) + f"\nNbr of trainable parameters: {self._n_trainable()}"


RESNET_BLOCKS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3), "resnet152": (3, 8, 36, 3),
                 "resnet14": (1, 1, 1, 1)}  # resnet14: shallow variant used by the batch-statistics parity test only


# ----------------------------------------------------------------------------------------------- holders
class _Holder(nn.Module):
    """Named container of parameter-holding children; never executed."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("seg_b200 modules are parameter holders; call the top-level model")


def _cbn(cin, cout, k, stride=1, dil=1, pad=None):
    if pad is None:
        pad = 0 if k == 1 else dil
    return nn.Conv2d(cin, cout, k, stride=stride, padding=pad, dilation=dil, bias=False), nn.BatchNorm2d(cout)


def _bottleneck(inplanes, planes, stride, dil, with_downsample):
    b = _Holder()
    b.conv1, b.bn1 = _cbn(inplanes, planes, 1)
    b.conv2, b.bn2 = _cbn(planes, planes, 3, stride, dil)
    b.conv3, b.bn3 = _cbn(planes, planes * 4, 1)
    b.relu = nn.ReLU(inplace=True)
    if with_downsample:
        c, n = _cbn(inplanes, planes * 4, 1, stride)
        b.downsample = nn.Sequential(c, n)
    else:
        b.downsample = None
    return b


def _res_layers(blocks, inplanes, plan):
    """plan: per layer (first-block stride, first-block dilation, other-block dilation), or (first-block stride, [dilation
    of every block]) for per-block rates such as HDC's (duc_hdc.py:78-103)."""
    layers = []
    for li, (n, planes) in enumerate(zip(blocks, (64, 128, 256, 512))):
        stride, *d = plan[li]
        dils = list(d[0]) if len(d) == 1 else [d[0]] + [d[1]] * (n - 1)
        assert len(dils) == n, f"layer{li + 1}: {len(dils)} dilations for {n} blocks"
        seq = []
        for b in range(n):
            seq.append(_bottleneck(inplanes, planes, stride if b == 0 else 1, dils[b], b == 0))
            inplanes = planes * 4
        layers.append(nn.Sequential(*seq))
    return layers


def _stem7(in_channels, stride=2):
    """torchvision ResNet stem holder: 7x7 conv (64) - BN - ReLU - 3x3/2 max-pool."""
    c, n = nn.Conv2d(in_channels, 64, 7, stride=stride, padding=3, bias=False), nn.BatchNorm2d(64)
    return nn.Sequential(c, n, nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2, padding=1))


def _deep_stem():
    """Deep stem holder (resnet.py:137-151): [3x3/2 conv-BN-ReLU, 3x3 conv-BN-ReLU, 3x3 conv to 128], its BN, ReLU, 3x3/2
    max-pool."""
    s1, n1 = _cbn(3, 64, 3, 2, 1)
    s2, n2 = _cbn(64, 64, 3, 1, 1)
    s3 = nn.Conv2d(64, 128, 3, stride=1, padding=1, bias=False)
    stem = nn.Sequential(s1, n1, nn.ReLU(inplace=True), s2, n2, nn.ReLU(inplace=True), s3)
    return nn.Sequential(stem, nn.BatchNorm2d(128), nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2, padding=1))


def _psp_module(m, bins, out):
    """_PSPModule holder (pspnet.py:11-38, upernet.py:9-38): per bin an adaptive average pool and a 1x1 conv-BN-ReLU to m // 4
    channels; the bottleneck, a 3x3 conv-BN-ReLU-Dropout2d(0.1) from the 2m-channel concat to `out` channels."""
    psp = _Holder()
    stages = []
    for b in bins:
        c, n = _cbn(m, m // 4, 1)
        stages.append(nn.Sequential(nn.AdaptiveAvgPool2d(output_size=b), c, n, nn.ReLU(inplace=True)))
    psp.stages = nn.ModuleList(stages)
    c, n = _cbn(m * 2, out, 3)
    psp.bottleneck = nn.Sequential(c, n, nn.ReLU(inplace=True), nn.Dropout2d(0.1))
    return psp


def _psp_branches(m, aux_in, num_classes):
    """PSPNet's (master_branch, auxiliary_branch) (pspnet.py:59-70): the PSP module (bins 1, 2, 3, 6) over the m-channel
    trunk output + a 1x1 classifier; a 3x3 conv-BN-ReLU-Dropout2d(0.1) over the aux_in-channel aux features + a 1x1
    classifier."""
    master = nn.Sequential(_psp_module(m, (1, 2, 3, 6), m // 4), nn.Conv2d(m // 4, num_classes, kernel_size=1))
    c, n = _cbn(aux_in, m // 4, 3)
    aux = nn.Sequential(c, n, nn.ReLU(inplace=True), nn.Dropout2d(0.1), nn.Conv2d(m // 4, num_classes, kernel_size=1))
    return master, aux


def _aspp_module(dilations):
    """ASSP holder (deeplabv3_plus.py:260-284, duc_hdc.py:126-155) over the 2048-channel trunk output: per dilation a
    256-channel conv-BN-ReLU branch (1x1 for the first, 3x3 dilated for the others), image pooling, and the 1x1
    conv-BN-ReLU-Dropout(0.5) over the concat."""
    a = _Holder()
    for i, d in enumerate(dilations, 1):
        c, n = _cbn(2048, 256, 1 if i == 1 else 3, 1, d)
        setattr(a, f"aspp{i}", nn.Sequential(c, n, nn.ReLU(inplace=True)))
    c, n = _cbn(2048, 256, 1)
    a.avg_pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), c, n, nn.ReLU(inplace=True))
    a.conv1, a.bn1 = _cbn(256 * (len(dilations) + 1), 256, 1)
    a.relu, a.dropout = nn.ReLU(inplace=True), nn.Dropout(0.5)
    return a


def _freeze(params):
    """freeze_backbone: the parameters stop receiving gradients."""
    for p in params:
        p.requires_grad = False


def _sepconv(cin, cout, stride, dil):
    """SeparableConv2d holder (deeplabv3_plus.py:70-86): depthwise 3x3 'same' conv -> BN -> pointwise 1x1."""
    s = _Holder()
    pad = dil if dil > 1 else 1
    s.conv1 = nn.Conv2d(cin, cin, 3, stride, padding=pad, dilation=dil, groups=cin, bias=False)
    s.bn = nn.BatchNorm2d(cin)
    s.pointwise = nn.Conv2d(cin, cout, 1, 1, bias=False)
    return s


def _xception_block(cin, cout, stride=1, dil=1, exit_flow=False, use_1st_relu=True):
    """Block holder (deeplabv3_plus.py:89-121) with the reference's child order / Sequential indices."""
    b = _Holder()
    if cin != cout or stride != 1:
        b.skip = nn.Conv2d(cin, cout, 1, stride=stride, bias=False)
        b.skipbn = nn.BatchNorm2d(cout)
    else:
        b.skip = None
    b.relu = nn.ReLU(inplace=True)
    units = [(cin, cin), (cin, cout), (cout, cout)] if exit_flow else [(cin, cout), (cout, cout), (cout, cout)]
    rep = []
    for i, (a, c) in enumerate(units):
        rep += [b.relu, _sepconv(a, c, stride if i == 2 else 1, dil), nn.BatchNorm2d(c)]
    if not use_1st_relu:
        rep = rep[1:]
    b.rep = nn.Sequential(*rep)
    b.use_1st_relu = use_1st_relu
    return b


def _xception_trunk(output_stride):
    """Aligned Xception holder (deeplabv3_plus.py:134-171)."""
    b3_s, mf_d, ef_d = (2, 1, (1, 2)) if output_stride == 16 else (1, 2, (2, 4))
    x = _Holder()
    x.conv1 = nn.Conv2d(3, 32, 3, 2, padding=1, bias=False)
    x.bn1 = nn.BatchNorm2d(32)
    x.relu = nn.ReLU(inplace=True)
    x.conv2 = nn.Conv2d(32, 64, 3, 1, padding=1, bias=False)
    x.bn2 = nn.BatchNorm2d(64)
    x.block1 = _xception_block(64, 128, stride=2, dil=1, use_1st_relu=False)
    x.block2 = _xception_block(128, 256, stride=2, dil=1)
    x.block3 = _xception_block(256, 728, stride=b3_s, dil=1)
    for i in range(16):
        setattr(x, f"block{i + 4}", _xception_block(728, 728, stride=1, dil=mf_d))
    x.block20 = _xception_block(728, 1024, stride=1, dil=ef_d[0], exit_flow=True)
    x.conv3, x.bn3 = _sepconv(1024, 1536, 1, ef_d[1]), nn.BatchNorm2d(1536)
    x.conv4, x.bn4 = _sepconv(1536, 1536, 1, ef_d[1]), nn.BatchNorm2d(1536)
    x.conv5, x.bn5 = _sepconv(1536, 2048, 1, ef_d[1]), nn.BatchNorm2d(2048)
    return x


def _init_like_reference_head(*mods):
    """utils/helpers.py:12-22 (initialize_weights): kaiming-normal convs (fan_in, relu), BN gamma=1, beta=1e-4."""
    for mod in mods:
        for m in mod.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight.data, nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1.0)
                m.bias.data.fill_(1e-4)


def _init_like_torchvision_trunk(*mods):
    for mod in mods:
        for m in mod.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)


def _init_like_resnet_s(*mods):
    """models/resnet.py:172-178: normal(0, sqrt(2/(k*k*cout))), BN 1/0."""
    for mod in mods:
        for m in mod.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()


def _check_pretrained(model, pretrained):
    """The reference's constructors default to pretrained=True and download ImageNet weights (resnet.py:21-27,
    deeplabv3_plus.py:172).  No network here: an explicit True raises; the default (None) — what a config that omits the key
    gets — initialises randomly like pretrained=False and says so once, instead of silently differing from the reference."""
    if pretrained:
        raise RuntimeError("pretrained weights need network access; load a state_dict instead")
    if pretrained is None:
        model.logger.warning("%s: the reference would download ImageNet weights here (pretrained defaults to True); this "
                             "build has no network and initialises randomly — load a state_dict, or pass pretrained=False "
                             "to silence this message", type(model).__name__)


# ----------------------------------------------------------------------------------------------- autograd bridge
class _EngineFn(torch.autograd.Function):
    """One autograd node for the whole model: forward = kernel tape, backward = tape replay.  With an initialised process
    group of more than one rank (one process per GPU) every parameter gradient is written into ONE flat fp32 buffer that is
    all-reduced (mean) inside backward — the replicas of an unmodified train.py stay identical, which is what the
    reference's nn.DataParallel wrapper guarantees (base/base_trainer.py:33-38)."""

    @staticmethod
    def forward(ctx, model, record, x, *params):
        world = model._dp_world() if record else 1
        views = flat = None
        if world > 1:
            flat = torch.zeros(sum(p.numel() for p in params if p.requires_grad), dtype=torch.float32, device=x.device)
            views, off = {}, 0
            for p in params:
                if p.requires_grad:
                    views[p] = flat[off:off + p.numel()].view(p.shape)
                    off += p.numel()
        outs, tape, heads = model._run(x, training=model.training, record=record, grads=views)
        ctx.tape, ctx.heads, ctx.params, ctx.flat, ctx.world = tape, heads, params, flat, world
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *douts):
        tape = ctx.tape
        if tape is None or not tape.record:
            raise RuntimeError("backward through a forward that ran without gradient recording")
        for head, dout in zip(ctx.heads, douts):
            if dout is None:
                continue
            head.logits_bwd(dout.contiguous().float())
        tape.backward()
        grads = tape.grads
        if ctx.flat is not None:
            from .comm import allreduce_mean_
            allreduce_mean_(ctx.flat, ctx.world)
            # pre-bound views hide which gradients the tape wrote: hand autograd only those (None otherwise, as at world 1)
            out = tuple(grads.get(p) if p in tape.touched else None for p in ctx.params)
        else:
            out = tuple(grads.get(p) for p in ctx.params)
        ctx.tape = None
        return (None, None, None) + out


class _GraphEntry:
    """Captured CUDA graphs of the plugin path for one (input shape, mode): `fwd` = weight packing + the forward tape up
    to the full-resolution fp32 NCHW logits, `bwd` = logits gradient -> every parameter gradient (one flat fp32 buffer).
    Both graphs allocate from one private memory pool, so the activations the forward graph writes are exactly what the
    backward graph reads; the ~1 000 kernel launches of a step become two `cudaGraphLaunch` calls."""

    def __init__(self, record, ptrs):
        self.record = record      # gradient recording (training step) or forward only (validation / inference)
        self.ptrs = ptrs          # data pointers of every parameter and buffer baked into the graphs
        self.pool = None
        self.fwd = self.bwd = None
        self.x = None
        self.outs = self.douts = None
        self.flat_grad = None
        self.param_slices = None  # per model.parameters() entry: (offset, numel, shape) into flat_grad, or None
        self.wt = None
        self.pending = False      # forward replayed, backward not yet: another forward would clobber the saved activations


class _GraphFn(torch.autograd.Function):
    """Autograd node of the graph-replayed plugin path (same contract as `_EngineFn`).  The returned logits alias the
    entry's static output buffer: like torch.cuda.make_graphed_callables, they are valid until the next forward."""

    @staticmethod
    def forward(ctx, entry, x, *params):
        entry.x.copy_(x, non_blocking=True)
        entry.fwd.replay()
        entry.pending = entry.record
        ctx.entry = entry
        if entry.record:
            outs = tuple(o.detach() for o in entry.outs)
        else:
            # forward-only entries (validation, inference.py's multi-scale / flip / sliding-window loops) hand out COPIES:
            # those callers keep one prediction alive across the next same-shape forward, which would overwrite a view
            # of the static buffer
            outs = tuple(o.detach().clone() for o in entry.outs)
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *douts):
        e = ctx.entry
        if e.bwd is None:
            raise RuntimeError("backward through a forward that ran without gradient recording")
        for s, d in zip(e.douts, douts):
            if d is None:
                s.zero_()
            else:
                s.copy_(d, non_blocking=True)
        e.bwd.replay()
        e.pending = False
        # hand autograd a private copy (ONE device copy of 4 bytes per parameter): AccumulateGrad may keep what it is
        # given, and the static buffer is rewritten by the next replay
        flat = e.flat_grad.clone()
        grads = tuple(None if sl is None else flat[sl[0]:sl[0] + sl[1]].view(sl[2]) for sl in e.param_slices)
        return (None, None) + grads


class _EngineModel(BaseModel):
    """Shared plumbing: spec cache, engine options, forward entry."""

    IM2COL_CONV = None  # the conv that reads the network input (NCHW fp32, any channel count) through the explicit im2col

    def __init__(self):
        super().__init__()
        self._specs = {}
        self._dwspecs = {}
        self.conv_impl = IMPL_AUTO
        self.engine_dropout = True    # set False to run train-mode parity with p = 0 (SURVEY.md §7)
        self.engine_seed = None       # None: derived from torch.initial_seed() and the data-parallel rank at first use
        self.bn_sync = None           # seg_b200.comm.SyncBNGroup for multi-GPU SyncBN
        self.use_sync_bn = False      # set by the overlay's convert_model (config "use_synch_bn"): attach a SyncBNGroup at the
                                      # first forward under a multi-rank process group
        self.dp_reduce = True         # all-reduce (mean) the gradients inside backward when world > 1
        self.syncbn_clamp_eps = True  # reproduce sync_batchnorm/batchnorm.py:145 when stats are synchronised
        self._step_ctr = None
        self._graphs_enabled = False
        self._graph_warmup = 2
        self._graph_entries = {}
        self._graph_seen = {}
        self._graph_max = 8           # captured (shape, mode) entries kept at most; further shapes run the eager tape
        self._flat_cache = None

    # ------------------------------------------------------------------ cached views of the module tree
    def _flat(self):
        """(parameters, parameters + buffers, BatchNorm modules) as flat lists.  Walking the module tree costs ~1.8 ms per
        call for DeepLab-R101 (680 tensors, ~500 modules) — more than the rest of a graph-replayed forward's host work —
        so the lists are built once and dropped whenever nn.Module re-creates tensors (`_apply`: .to / .cuda / .half)."""
        c = self._flat_cache
        if c is None:
            params = list(self.parameters())
            c = (params, params + list(self.buffers()), [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)])
            self._flat_cache = c
        return c

    def invalidate_caches(self):
        """Call after changing the module tree by hand (adding / replacing sub-modules or parameters)."""
        self._flat_cache = None
        self._specs, self._dwspecs = {}, {}
        self.release_graphs()

    def _apply(self, fn, *args, **kwargs):
        if getattr(self, "_graph_entries", None) is not None:
            self._flat_cache = None
            self.release_graphs()
        return super()._apply(fn, *args, **kwargs)

    def train(self, mode=True):
        # the trainer calls train() / eval() every epoch: re-walk the tree then, so a module swapped in by hand
        # (e.g. convert_model after construction) is picked up at the latest at the next epoch boundary
        if getattr(self, "_graph_entries", None) is not None:
            self._flat_cache = None
        return super().train(mode)

    # ------------------------------------------------------------------ CUDA-graph replay of the plugin path
    def cuda_graphs(self, enabled=True, warmup=2):
        """Opt in to graph replay of `model(x)` / `loss.backward()`: the first `warmup` calls with a given input shape
        and mode run eagerly (they are real steps and double as allocator / tensor-map warm-up), the next one captures
        the forward and backward tapes once, later calls replay them.  Contract (that of
        torch.cuda.make_graphed_callables): the returned logits live in a static buffer that the next forward of the
        same shape overwrites; one backward per forward (a forward issued while a backward is outstanding runs eagerly).
        At most `_graph_max` (8) distinct (shape, mode) combinations are captured — each owns a memory pool the size of
        the step's activations; others keep running the eager tape."""
        self._graphs_enabled = bool(enabled)
        self._graph_warmup = int(warmup)
        if not enabled:
            self.release_graphs()
        return self

    def release_graphs(self):
        if self._graph_entries:
            torch.cuda.synchronize()
            self._graph_entries = {}
            torch.cuda.synchronize()
        self._graph_seen = {}

    def _graph_lookup(self, x, record):
        _, tensors, bns = self._flat()
        bn_train = sum(1 for m in bns if m.training)
        key = (tuple(x.shape), x.device.index, self.training, bool(record), bn_train, bool(self.engine_dropout), self.bn_sync is not None,
               self._dp_world())
        ptrs = tuple(t.data_ptr() for t in tensors)
        e = self._graph_entries.get(key)
        if e is not None and e.ptrs != ptrs:  # a parameter / buffer was re-allocated (model.to(...), .half(), ...)
            torch.cuda.synchronize()
            del self._graph_entries[key]
            e = None
            self._graph_seen[key] = 0
        if e is None:
            n = self._graph_seen.get(key, 0)
            self._graph_seen[key] = n + 1
            if n < self._graph_warmup or len(self._graph_entries) >= self._graph_max:
                return None  # every entry owns a private memory pool (the step's activations): bound their number
            e = _GraphEntry(bool(record), ptrs)
            try:
                self._capture(e, x)
            except Exception:
                self._graphs_enabled = False  # do not retry every step; the caller sees the error
                raise
            self._graph_entries[key] = e
        if e.pending:
            # a recorded forward whose backward never ran (skipped step, exception, probe call): run THIS call on the eager
            # tape (the outstanding backward, if it still comes, needs the saved activations) and re-arm the entry
            e.pending = False
            if not getattr(self, "_graph_pending_warned", False):
                self._graph_pending_warned = True
                self.logger.warning("seg_b200: forward issued while a graph-replayed backward was outstanding; this call runs eagerly")
            return None
        return e

    @torch.no_grad()
    def _capture(self, e, x):
        """Capture the forward tape and (when recording) the backward tape of one step into two graphs sharing a pool."""
        from .train import WeightTables
        dev = x.device
        params = self._flat()[0]
        e.x = x.detach().contiguous().float().clone()
        views = None
        if e.record:
            total = sum(p.numel() for p in params if p.requires_grad)
            e.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
            views, slices, off = {}, [], 0
            for p in params:
                if not p.requires_grad:
                    slices.append(None)
                    continue
                views[p] = e.flat_grad[off:off + p.numel()].view(p.shape)
                slices.append((off, p.numel(), tuple(p.shape)))
                off += p.numel()
        e.wt = WeightTables(self, views, dev)
        e.pool = torch.cuda.graph_pool_handle()
        torch.cuda.synchronize()
        multi = torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1
        mode = "thread_local" if multi else "global"  # NCCL's watchdog thread polls events while we capture
        if multi and (self.bn_sync is not None or self.dp_reduce):
            torch.distributed.barrier()  # every rank has finished its eager exchanges before anyone captures
        fwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(fwd, pool=e.pool, capture_error_mode=mode):
            e.wt.pack()
            outs, tape, heads = self._run(e.x, training=self.training, record=e.record, tables=e.wt, grads=views)
        e.outs = outs
        if e.record:
            e.douts = [torch.zeros_like(o) for o in outs]
            torch.cuda.synchronize()
            bwd = torch.cuda.CUDAGraph()
            with torch.cuda.graph(bwd, pool=e.pool, capture_error_mode=mode):
                e.flat_grad.zero_()
                e.wt.zero_wgrads()
                for head, d in zip(heads, e.douts):
                    head.logits_bwd(d)
                tape.backward()
                e.wt.unpack()
                if self._dp_world() > 1:  # the gradient exchange is part of the captured backward (NCCL kernels replay)
                    from .comm import allreduce_mean_
                    allreduce_mean_(e.flat_grad, self._dp_world())
            e.bwd = bwd
            # parameters the tape never wrote a gradient for get None, as on the eager path
            e.param_slices = [sl if (sl is not None and p in tape.touched) else None for p, sl in zip(params, slices)]
        e.fwd = fwd
        torch.cuda.synchronize()

    def _spec(self, name, module):
        s = self._specs.get(name)
        if s is None or s.m is not module:
            s = ConvSpec(name, module, explicit_im2col=(name == self.IM2COL_CONV))
            self._specs[name] = s
        return s

    def all_conv_specs(self):
        """ConvSpec of every dense nn.Conv2d / nn.ConvTranspose2d holder (names = module paths, as used by the forward code)."""
        return [self._spec(n, m) for n, m in self.named_modules()
                if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)) and m.groups == 1]

    def all_dw_specs(self):
        return [self._dwspec(n, m) for n, m in self.named_modules() if isinstance(m, nn.Conv2d) and m.groups > 1]

    def _dwspec(self, name, module):
        s = self._dwspecs.get(name)
        if s is None or s.m is not module:
            s = DwSpec(name, module)
            self._dwspecs[name] = s
        return s

    def _sep_unit(self, tape, x, prefix, sep, bn_after, relu_after, res=None):
        """relu'd input -> depthwise -> BN -> pointwise -> BN (+res) (+ReLU of the NEXT unit, fused here)."""
        y, st = tape.dwconv(x, self._dwspec(prefix + ".conv1", sep.conv1), want_stats=True)
        a = tape.bn_act(y, sep.bn, st, relu=False)
        y2, st2 = tape.conv(a, self._spec(prefix + ".pointwise", sep.pointwise), want_stats=True)
        return tape.bn_act(y2, bn_after, st2, relu=relu_after, res=res)

    def _xblock(self, tape, x, prefix, blk, relu_out):
        """Xception Block (deeplabv3_plus.py:123-132).  `x` must already carry the block's leading in-place ReLU (every
        block but block1); `relu_out` fuses the NEXT block's leading ReLU — which, being in place, is also what that
        block's skip branch sees (SURVEY.md App. C.1)."""
        mods = list(blk.rep.named_children())
        units = [(i, m) for i, m in mods if isinstance(m, _Holder)]
        bns = {int(i): m for i, m in mods if isinstance(m, nn.BatchNorm2d)}
        skip = x
        if blk.skip is not None:
            skip = self._cbr(tape, x, prefix + "skip", blk.skip, blk.skipbn, relu=False)
        h = x
        for k, (idx, sep) in enumerate(units):
            last = k == len(units) - 1
            h = self._sep_unit(tape, h, f"{prefix}rep.{idx}", sep, bns[int(idx) + 1], relu_after=(relu_out if last else True),
                               res=skip if last else None)
        return h

    def _new_tape(self, training, record):
        ctr = None
        if training:
            dev = next(self.parameters()).device
            if self._step_ctr is None or self._step_ctr.device != dev:
                # starts from the first BatchNorm's num_batches_tracked (a checkpointed buffer): a resumed run continues
                # the dropout-mask sequence instead of repeating it from step 0
                bns = self._flat()[2]
                start = bns[0].num_batches_tracked.detach().reshape(1).to(dev, torch.int64) if bns else None
                self._step_ctr = start.clone() if start is not None else torch.zeros(1, dtype=torch.int64, device=dev)
            ctr = self._step_ctr
            ops.counter_add(ctr, 1)  # device-side: stays correct when the step is replayed from a CUDA graph
        return Tape(training, record=record, impl=self.conv_impl, dropout=self.engine_dropout, seed=self._seed(),
                    sync=self.bn_sync, clamp_eps=self.syncbn_clamp_eps, step_ctr=ctr,
                    arena_floats=getattr(self, "_arena_floats", 0) if training else 0, owner=self)

    def _seed(self):
        """Dropout seed: follows torch.manual_seed and differs per data-parallel rank (nn.Dropout under DataParallel draws
        independent masks per replica); the per-step variation comes from the device-side step counter."""
        if self.engine_seed is None:
            rank = torch.distributed.get_rank() if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 0
            self.engine_seed = (int(torch.initial_seed()) * 2654435761 + rank * 0x9E3779B1) & 0x7FFFFFFF
        return self.engine_seed

    def _cbr(self, tape, x, name, conv, bn, relu=True, res=None, out=None, drop_p=0.0, drop_channelwise=False):
        y, st = tape.conv(x, self._spec(name, conv), want_stats=True)
        return tape.bn_act(y, bn, st, relu=relu, res=res, out=out, drop_p=drop_p, drop_channelwise=drop_channelwise)

    def _block(self, tape, x, prefix, blk, out=None):
        a = self._cbr(tape, x, prefix + "conv1", blk.conv1, blk.bn1)
        a = self._cbr(tape, a, prefix + "conv2", blk.conv2, blk.bn2)
        r = x
        if blk.downsample is not None:
            r = self._cbr(tape, x, prefix + "downsample.0", blk.downsample[0], blk.downsample[1], relu=False)
        return self._cbr(tape, a, prefix + "conv3", blk.conv3, blk.bn3, relu=True, res=r, out=out)

    def _stem(self, tape, x, name, stem):
        """A ResNet stem holder (`_stem7` or `_deep_stem`) at `name`: its conv-BN-ReLU units, then the 3x3/2 max-pool."""
        if isinstance(stem[0], nn.Sequential):  # deep stem: the third conv's BN is the outer holder's
            s = stem[0]
            for i, bn in ((0, s[1]), (3, s[4]), (6, stem[1])):
                x = self._cbr(tape, x, f"{name}.0.{i}", s[i], bn)
        else:
            x = self._cbr(tape, x, f"{name}.0", stem[0], stem[1])
        return tape.maxpool(x)

    def _trunk(self, tape, x, prefix, stem):
        """ResNet trunk: the stem holder `stem` and layer1..4, attributes of the module at `prefix` ("" = the model); returns
        the four layer outputs."""
        owner = self.get_submodule(prefix.rstrip(".")) if prefix else self
        a = self._stem(tape, x, prefix + stem, getattr(owner, stem))
        feats = []
        for li in (1, 2, 3, 4):
            for bi, blk in enumerate(getattr(owner, f"layer{li}")):
                a = self._block(tape, a, f"{prefix}layer{li}.{bi}.", blk)
            feats.append(a)
        return feats

    def _ppm(self, tape, a, psp, prefix, cat=None):
        """_PSPModule.forward (pspnet.py:31-38, upernet.py:31-38) of the `_psp_module` holder `psp` at `prefix`: cat([a, one
        stage per bin]) -> bottleneck; returns the bottleneck's output.  a: the trunk output (m channels; stages of m // 4).
        cat: a `dense_buffer` of 2m channels whose first m the trunk wrote in place (PSPDenseNet's block4); otherwise the
        concat is allocated here and a, which is also the residual stream's tensor, is copied into slice 0."""
        N, Hf, Wf, m = a.t.shape
        q = m // 4
        if cat is None:
            cat, sl = tape.concat(N, Hf, Wf, [m, q, q, q, q], a.t.device)
            feats = tape.copy_into(a, sl[0])
        else:
            sl = [cat.t[..., :m]] + [cat.t[..., m + i * q:m + (i + 1) * q] for i in range(4)]
            feats = a
        br = [feats]
        for i, st in enumerate(psp.stages):
            p = tape.avgpool(a, st[0].output_size)
            p = self._cbr(tape, p, f"{prefix}.stages.{i}.1", st[1], st[2])
            br.append(tape.bilinear(p, Hf, Wf, True, out=sl[i + 1]))
        tape.bind_slices(cat, br)
        b = psp.bottleneck
        return self._cbr(tape, cat, f"{prefix}.bottleneck.0", b[0], b[1], drop_p=b[3].p, drop_channelwise=True)

    def _aspp(self, tape, a):
        """ASSP.forward (deeplabv3_plus.py:286-297, duc_hdc.py:157-174) of the `_aspp_module` holder `ASSP`: every dilated
        branch and the image pooling written straight into one concat buffer, then the 1x1 fusion conv."""
        N, Hf, Wf = a.t.shape[0], a.t.shape[1], a.t.shape[2]
        A = self.ASSP
        branches = [seq for name, seq in A.named_children() if name.startswith("aspp")]
        cat, sl = tape.concat(N, Hf, Wf, [256] * (len(branches) + 1), a.t.device)
        br = [self._cbr(tape, a, f"ASSP.aspp{i + 1}.0", seq[0], seq[1], out=sl[i]) for i, seq in enumerate(branches)]
        g = tape.avgpool(a, 1)
        g = self._cbr(tape, g, "ASSP.avg_pool.1", A.avg_pool[1], A.avg_pool[2])
        br.append(tape.bilinear(g, Hf, Wf, True, out=sl[-1]))
        tape.bind_slices(cat, br)
        return self._cbr(tape, cat, "ASSP.conv1", A.conv1, A.bn1, drop_p=A.dropout.p)

    def _finish(self, tape):
        # one count per normalisation: a BN applied twice in a step (PSPDenseNet's block0.4) advances by 2, as the reference's
        counts = {}
        for m in tape.bn_modules:
            counts[m] = counts.get(m, 0) + 1
        for k in sorted(set(counts.values())):
            torch._foreach_add_([m.num_batches_tracked for m, c in counts.items() if c == k], k)

    def _dp_world(self):
        """Data-parallel replicas taking part in this model's backward (1 = no exchange)."""
        if not self.dp_reduce:
            return 1
        from .comm import dp_world
        return dp_world()

    def _attach_sync_bn(self):
        """config['use_synch_bn'] (base/base_trainer.py:33-35 -> the overlay's convert_model) under torchrun: BatchNorm
        statistics are exchanged over NVLink peer memory (sync_batchnorm/batchnorm.py:105-145 semantics, clamp(var, eps))."""
        from . import comm
        if self.use_sync_bn and self.bn_sync is None and comm.dp_world() > 1:
            self.bn_sync = comm.SyncBNGroup()
            self.release_graphs()

    def _check_input(self, x):
        if not x.is_cuda:
            raise RuntimeError("seg_b200 models run on an H100 only; there is no CPU / eager fallback")
        require_device()

    def forward(self, x):
        self._check_input(x)
        if self.use_sync_bn and self.bn_sync is None:
            self._attach_sync_bn()
        params = self._flat()[0]
        record = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        if self._graphs_enabled:
            e = self._graph_lookup(x, record)
            if e is not None:
                return _GraphFn.apply(e, x, *params)
        return _EngineFn.apply(self, record, x, *params)

    def _run(self, x, training, record, tables=None, grads=None):
        x = x.contiguous().float()
        tape = self._new_tape(training, record)
        if tables is not None:  # graph capture: persistent packed weights / packed weight-gradient accumulators
            tape.packed_override, tape.dw_buffers = tables.packed_bufs, tables.dw_bufs
        if grads is not None:
            tape.grads = dict(grads)  # pre-bound views: every parameter gradient lands in one flat buffer
        heads = self._forward_heads(tape, x)
        outs = tuple(h.logits() for h in heads)
        self._finish(tape)
        return outs, tape, heads

    def freeze_bn(self):
        for module in self.modules():
            if isinstance(module, nn.BatchNorm2d):
                module.eval()


# ----------------------------------------------------------------------------------------------- DeepLabV3+
class DeepLab(_EngineModel):
    """DeepLabV3+ with a (dilated) torchvision-style ResNet trunk — replaces models/deeplabv3_plus.py:336-377."""

    def __init__(self, num_classes, in_channels=3, backbone="xception", pretrained=None, output_stride=16,
                 freeze_bn=False, freeze_backbone=False, **_):
        super().__init__()
        if backbone != "xception" and backbone not in RESNET_BLOCKS:
            raise NotImplementedError(f"seg_b200.DeepLab: backbone {backbone!r} not built (xception, resnet50/101/152 are)")
        _check_pretrained(self, pretrained)
        assert output_stride in (8, 16)
        self.num_classes, self.output_stride, self.backbone_name = num_classes, output_stride, backbone
        if backbone == "xception":
            self._build_heads(num_classes, output_stride, low_level_channels=128)
            self.backbone = _xception_trunk(output_stride)
            # keep the reference's registration order: backbone, ASSP, decoder
            assp, dec = self.ASSP, self.decoder
            del self.ASSP, self.decoder
            self.ASSP, self.decoder = assp, dec
            _init_like_reference_head(self.backbone, self.ASSP, self.decoder)
        else:
            # deeplabv3_plus.py:35-53: os16 -> layer3 stride 2, layer4 every conv2 d=2 ; os8 -> layer3 d=2, layer4 d=4
            if output_stride == 16:
                plan = [(1, 1, 1), (2, 1, 1), (2, 1, 1), (1, 2, 2)]
            else:
                plan = [(1, 1, 1), (2, 1, 1), (1, 2, 2), (1, 4, 4)]
            bb = _Holder()
            bb.layer0 = _stem7(in_channels)
            bb.layer1, bb.layer2, bb.layer3, bb.layer4 = _res_layers(RESNET_BLOCKS[backbone], 64, plan)
            self.backbone = bb
            self._build_heads(num_classes, output_stride, low_level_channels=256)
            _init_like_torchvision_trunk(bb.layer1, bb.layer2, bb.layer3, bb.layer4)
            _init_like_reference_head(bb.layer0, self.ASSP, self.decoder)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(self.backbone.parameters())

    def _build_heads(self, num_classes, output_stride, low_level_channels):
        self.ASSP = _aspp_module((1, 6, 12, 18) if output_stride == 16 else (1, 12, 24, 36))
        d = _Holder()
        d.conv1, d.bn1 = _cbn(low_level_channels, 48, 1)
        d.relu = nn.ReLU(inplace=True)
        c1, n1 = _cbn(48 + 256, 256, 3)
        c2, n2 = _cbn(256, 256, 3)
        d.output = nn.Sequential(c1, n1, nn.ReLU(inplace=True), c2, n2, nn.ReLU(inplace=True), nn.Dropout(0.1),
                                 nn.Conv2d(256, num_classes, 1, stride=1))
        self.decoder = d

    # ---- engine forward: returns the stride-4 fp32 logits Act (NHWC) ----
    def _trunk_xception(self, tape, x):
        """Xception.forward (deeplabv3_plus.py:201-247); low-level features = block1 output BEFORE the ReLU."""
        bb = self.backbone
        a = self._cbr(tape, x, "backbone.conv1", bb.conv1, bb.bn1)
        a = self._cbr(tape, a, "backbone.conv2", bb.conv2, bb.bn2, relu=False)
        low = self._xblock(tape, a, "backbone.block1.", bb.block1, relu_out=False)
        a = tape.relu(low)
        for i in range(2, 21):
            a = self._xblock(tape, a, f"backbone.block{i}.", getattr(bb, f"block{i}"), relu_out=True)
        for n in (3, 4, 5):
            a = self._sep_unit(tape, a, f"backbone.conv{n}", getattr(bb, f"conv{n}"), getattr(bb, f"bn{n}"), relu_after=True)
        return a, low

    def _decoder(self, tape, f, low):
        """Decoder.forward (deeplabv3_plus.py:323-330): concat order (low-level 48, upsampled 256); returns the fp32
        stride-4 logits Act."""
        D = self.decoder
        N, Hl, Wl = low.t.shape[0], low.t.shape[1], low.t.shape[2]
        cat2, sl2 = tape.concat(N, Hl, Wl, [48, 256], low.t.device)
        l48 = self._cbr(tape, low, "decoder.conv1", D.conv1, D.bn1, out=sl2[0])
        up = tape.bilinear(f, Hl, Wl, True, out=sl2[1])
        tape.bind_slices(cat2, [l48, up])
        y = self._cbr(tape, cat2, "decoder.output.0", D.output[0], D.output[1])
        y = self._cbr(tape, y, "decoder.output.3", D.output[3], D.output[4], drop_p=D.output[6].p)
        lo, _ = tape.conv(y, self._spec("decoder.output.7", D.output[7]), out_dtype=torch.float32)
        return lo

    def _features(self, tape, x):
        if self.backbone_name == "xception":
            a, low = self._trunk_xception(tape, x)
        else:
            low, _, _, a = self._trunk(tape, x, "backbone.", "layer0")
        return self._decoder(tape, self._aspp(tape, a), low)

    def _forward_heads(self, tape, x):
        """[head of the stride-4 fp32 logits]  (deeplabv3_plus.py:361: align_corners=True)"""
        return [BilinearHead(self._features(tape, x), True, x.shape[2], x.shape[3])]

    def get_backbone_params(self):
        return self.backbone.parameters()

    def get_decoder_params(self):
        return chain(self.ASSP.parameters(), self.decoder.parameters())


# ----------------------------------------------------------------------------------------------- PSPNet
class PSPNet(_EngineModel):
    """PSPNet over the deep-stem dilated ResNet — replaces models/pspnet.py:41-105 + models/resnet.py:124-212."""

    def __init__(self, num_classes, in_channels=3, backbone="resnet152", pretrained=None, use_aux=True, freeze_bn=False,
                 freeze_backbone=False, **_):
        super().__init__()
        if backbone not in RESNET_BLOCKS:
            raise NotImplementedError(f"seg_b200.PSPNet: backbone {backbone!r} not built")
        _check_pretrained(self, pretrained)
        if in_channels != 3:
            raise NotImplementedError("in_channels != 3 swaps the deep stem for a 7x7 conv (pspnet.py:50-51); not built")
        self.num_classes, self.use_aux = num_classes, use_aux
        self.initial = _deep_stem()
        # resnet.py:154-163,190-210: layer3 = [d1, d2, ...], layer4 = [d2, d4, ...], all stride 1 (output stride 8)
        plan = [(1, 1, 1), (2, 1, 1), (1, 1, 2), (1, 2, 4)]
        self.layer1, self.layer2, self.layer3, self.layer4 = _res_layers(RESNET_BLOCKS[backbone], 128, plan)
        self.master_branch, self.auxiliary_branch = _psp_branches(2048, 1024, num_classes)
        _init_like_resnet_s(self.initial, self.layer1, self.layer2, self.layer3, self.layer4)
        _init_like_reference_head(self.master_branch, self.auxiliary_branch)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(self.get_backbone_params())

    def _forward_heads(self, tape, x):
        _, _, x_aux, a = self._trunk(tape, x, "", "initial")
        lo = self._psp_head(tape, a)
        H, W = x.shape[2], x.shape[3]
        heads = [BilinearHead(lo, False, H, W)]  # pspnet.py:86,91: F.interpolate default align_corners=False; the crop is a no-op
        if self.training and self.use_aux:
            ab = self.auxiliary_branch
            ya = self._cbr(tape, x_aux, "auxiliary_branch.0", ab[0], ab[1], drop_p=ab[3].p, drop_channelwise=True)
            la, _ = tape.conv(ya, self._spec("auxiliary_branch.4", ab[4]), out_dtype=torch.float32)
            heads.append(BilinearHead(la, False, H, W))
        return heads

    def _psp_head(self, tape, a, cat=None):
        """master_branch (pspnet.py:85): the PSP module + the classifier; returns the fp32 stride-8 logits Act.  a, cat: as
        `_ppm`'s."""
        y = self._ppm(tape, a, self.master_branch[0], "master_branch.0", cat=cat)
        lo, _ = tape.conv(y, self._spec("master_branch.1", self.master_branch[1]), out_dtype=torch.float32)
        return lo

    def get_backbone_params(self):
        return chain(self.initial.parameters(), self.layer1.parameters(), self.layer2.parameters(), self.layer3.parameters(),
                     self.layer4.parameters())

    def get_decoder_params(self):
        return chain(self.master_branch.parameters(), self.auxiliary_branch.parameters())


# ----------------------------------------------------------------------------------------------- UperNet
class UperNet(_EngineModel):
    """UperNet (object path) — replaces models/upernet.py:119-154: torchvision-ResNet trunk returning four feature maps
    (:40-87, output stride 16), PSPModule bins {1,2,4,6} (:9-38), FPN_fuse (:92-117), 3x3 head, bilinear(align_corners=
    False) to the input size.  Quirks kept: ONE smooth conv shared by the three FPN levels (three aliased state_dict
    entries), non-cumulative top-down path, laterals / smooth / head carry a bias, conv_fusion does not.
    (The reference constructor itself raises NameError: freeze_backbone, upernet.py:133 — here the argument works.)"""

    def __init__(self, num_classes, in_channels=3, backbone="resnet101", pretrained=None, use_aux=True, fpn_out=256,
                 freeze_bn=False, freeze_backbone=False, **_):
        super().__init__()
        if backbone not in RESNET_BLOCKS:
            raise NotImplementedError(f"seg_b200.UperNet: backbone {backbone!r} not built (bottleneck ResNets are)")
        _check_pretrained(self, pretrained)
        self.num_classes = num_classes
        bb = _Holder()
        bb.initial = _stem7(in_channels)
        bb.layer1, bb.layer2, bb.layer3, bb.layer4 = _res_layers(RESNET_BLOCKS[backbone], 64, [(1, 1, 1), (2, 1, 1), (2, 1, 1), (1, 2, 2)])
        self.backbone = bb
        feats = [256, 512, 1024, 2048]
        self.PPN = _psp_module(feats[-1], (1, 2, 4, 6), feats[-1])
        fpn = _Holder()
        fpn.conv1x1 = nn.ModuleList([nn.Conv2d(f, fpn_out, kernel_size=1) for f in feats[1:]])
        fpn.smooth_conv = nn.ModuleList([nn.Conv2d(fpn_out, fpn_out, kernel_size=3, padding=1)] * (len(feats) - 1))
        c, n = _cbn(len(feats) * fpn_out, fpn_out, 3)
        fpn.conv_fusion = nn.Sequential(c, n, nn.ReLU(inplace=True))
        self.FPN = fpn
        self.head = nn.Conv2d(fpn_out, num_classes, kernel_size=3, padding=1)
        _init_like_torchvision_trunk(bb.layer1, bb.layer2, bb.layer3, bb.layer4)
        _init_like_reference_head(bb.initial)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(self.backbone.parameters())

    def _forward_heads(self, tape, x):
        N = x.shape[0]
        feats = self._trunk(tape, x, "backbone.", "initial")
        feats[-1] = self._ppm(tape, feats[-1], self.PPN, "PPN")  # PPN on the last feature map (upernet.py:31-38)
        # ---- FPN_fuse (upernet.py:103-117) ----
        F_ = self.FPN
        lat = [feats[0]]
        for i in range(3):
            y, _ = tape.conv(feats[i + 1], self._spec(f"FPN.conv1x1.{i}", F_.conv1x1[i]))
            lat.append(y)
        smooth = self._spec("FPN.smooth_conv.0", F_.smooth_conv[0])  # one shared conv, applied three times
        P = []
        for i in (3, 2, 1):
            u = tape.up_add(lat[i], lat[i - 1])
            y, _ = tape.conv(u, smooth)
            P.append(y)
        P = list(reversed(P)) + [lat[-1]]
        H1, W1 = P[0].t.shape[1], P[0].t.shape[2]
        cat2, sl2 = tape.concat(N, H1, W1, [256] * 4, x.device)
        parts = [tape.copy_into(P[0], sl2[0])]
        for j in (1, 2, 3):
            parts.append(tape.bilinear(P[j], H1, W1, True, out=sl2[j]))
        tape.bind_slices(cat2, parts)
        y = self._cbr(tape, cat2, "FPN.conv_fusion.0", F_.conv_fusion[0], F_.conv_fusion[1])
        lo, _ = tape.conv(y, self._spec("head", self.head), out_dtype=torch.float32)
        return [BilinearHead(lo, False, x.shape[2], x.shape[3])]  # upernet.py:143: F.interpolate default align_corners=False

    def get_backbone_params(self):
        return self.backbone.parameters()

    def get_decoder_params(self):
        return chain(self.PPN.parameters(), self.FPN.parameters(), self.head.parameters())


# ----------------------------------------------------------------------------------------------- DeepLab_DUC_HDC
def _duc(cin, cout, r):
    """DUC holder (duc_hdc.py:15-31): 1x1 conv to cout*r*r channels without bias, BN, ReLU, PixelShuffle(r)."""
    d = _Holder()
    d.conv = nn.Conv2d(cin, cout * r * r, 1, bias=False)
    d.bn = nn.BatchNorm2d(cout * r * r)
    d.relu = nn.ReLU(inplace=True)
    d.pixl_shf = nn.PixelShuffle(upscale_factor=r)
    return d


def _icnr_(conv, r):
    """duc_hdc.py:33-49 (ICNR): the r*r output channels of one shuffle group share one kaiming-normal kernel."""
    o, i, kh, kw = conv.weight.shape
    sub = nn.init.kaiming_normal_(torch.empty(o // (r * r), i, kh, kw))
    conv.weight.data.copy_(sub.repeat_interleave(r * r, dim=0))


class DeepLab_DUC_HDC(_EngineModel):
    """DeepLab v3+ with HDC dilations and DUC upsampling — replaces models/duc_hdc.py:214-245: a ResNet-101 trunk at output
    stride 8 (layer3 / layer4 at stride 1 with per-block rates [1,2,3]*7+[2,2] and [3,4,5]; output_stride=4 also drops the
    stem conv's stride), a six-branch ASPP + image pooling, a decoder whose x2 upsampling is DUC (1x1 conv, BN, ReLU,
    PixelShuffle(2), cropped to the low-level size) and DUC_out = DUC(C, C, 4): the model returns the ReLU'd, pixel-shuffled
    [N, C, 4*Hl, 4*Wl] scores (Hl, Wl: layer1 size; a 65x65 input gives 68x68, as in the reference).
    Quirks kept: ICNR init on DUC_out.conv only (the decoder's initialize_weights overwrites decoder.DUC.conv).
    (The reference constructor itself raises NameError: freeze_backbone, duc_hdc.py:225 — here the argument works.)"""

    def __init__(self, num_classes, in_channels=3, pretrained=None, output_stride=8, freeze_bn=False, freeze_backbone=False, **_):
        super().__init__()
        _check_pretrained(self, pretrained)
        assert output_stride in (4, 8), "Only output strides of 8 or 16 are suported"
        self.num_classes, self.output_stride = num_classes, output_stride
        bb = _Holder()
        bb.layer0 = _stem7(in_channels, stride=2 if output_stride == 8 else 1)
        plan = [(1, [1] * 3), (2, [1] * 4), (1, [1, 2, 3] * 7 + [2, 2]), (1, [3, 4, 5])]
        bb.layer1, bb.layer2, bb.layer3, bb.layer4 = _res_layers(RESNET_BLOCKS["resnet101"], 64, plan)
        self.backbone = bb
        self.ASSP = _aspp_module((1, 6, 12, 18, 24, 36))
        d = _Holder()
        d.conv1, d.bn1 = _cbn(256, 48, 1)
        d.relu = nn.ReLU(inplace=True)
        d.DUC = _duc(256, 256, 2)
        c1, n1 = _cbn(48 + 256, 256, 3)
        c2, n2 = _cbn(256, 256, 3)
        d.output = nn.Sequential(c1, n1, nn.ReLU(inplace=True), c2, n2, nn.ReLU(inplace=True), nn.Dropout(0.1),
                                 nn.Conv2d(256, num_classes, 1, stride=1))
        self.decoder = d
        self.DUC_out = _duc(num_classes, num_classes, 4)
        _init_like_torchvision_trunk(bb.layer1, bb.layer2, bb.layer3, bb.layer4)
        _init_like_reference_head(bb.layer0, self.ASSP, self.decoder, self.DUC_out)
        _icnr_(self.DUC_out.conv, 4)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(self.backbone.parameters())

    def _decoder(self, tape, f, low):
        """Decoder.forward (duc_hdc.py:200-208): the DUC output is shuffled and cropped straight into the concat buffer
        (low-level 48, upsampled 256); returns the bf16 class scores Act (pitch padded to 8 channels for DUC_out's im2col)."""
        D = self.decoder
        N, Hl, Wl = low.t.shape[0], low.t.shape[1], low.t.shape[2]
        cat, sl = tape.concat(N, Hl, Wl, [48, 256], low.t.device)
        l48 = self._cbr(tape, low, "decoder.conv1", D.conv1, D.bn1, out=sl[0])
        u = self._cbr(tape, f, "decoder.DUC.conv", D.DUC.conv, D.DUC.bn)
        up = tape.pixel_shuffle(u, 2, out=sl[1], crop=(Hl, Wl))
        tape.bind_slices(cat, [l48, up])
        y = self._cbr(tape, cat, "decoder.output.0", D.output[0], D.output[1])
        y = self._cbr(tape, y, "decoder.output.3", D.output[3], D.output[4], drop_p=D.output[6].p)
        C = self.num_classes
        buf = torch.empty((N, Hl, Wl, (C + 7) // 8 * 8), dtype=y.t.dtype, device=y.t.device)[..., :C]
        lo, _ = tape.conv(y, self._spec("decoder.output.7", D.output[7]), out=buf)
        return lo

    def _forward_heads(self, tape, x):
        low, _, _, a = self._trunk(tape, x, "backbone.", "layer0")
        y = self._decoder(tape, self._aspp(tape, a), low)
        z = self._cbr(tape, y, "DUC_out.conv", self.DUC_out.conv, self.DUC_out.bn)
        return [ShuffleHead(z, 4)]

    def get_backbone_params(self):
        return self.backbone.parameters()

    def get_decoder_params(self):
        return chain(self.ASSP.parameters(), self.decoder.parameters(), self.DUC_out.parameters())


# ----------------------------------------------------------------------------------------------- UNetResnet
class UNetResnet(_EngineModel):
    """U-Net decoder over the deep-stem dilated ResNet — replaces models/unet.py:126-209.  The trunk is PSPNet's (`initial`
    = deep stem + bn1 + ReLU + max-pool, layer3 / layer4 at stride 1 with dilations 2 / 4: x2, x3 and x4 are all at 1/8).
    Decoder: convs WITH bias and no BN / ReLU, ConvTranspose2d(4, 2, 1) x2 upsamplings, bilinear(align_corners=True)
    resamples to each skip's size, concat (upsampled, skip), and conv7 (1x1, no bias) on a map at input resolution: the
    model returns full-resolution logits for any input size (a 65x65 input reaches 68x68 after upconv5 and is resampled).
    Quirks kept: initialize_weights runs over the whole model (trunk included: kaiming-normal convs, BN gamma 1 / beta
    1e-4); conv biases and the ConvTranspose2d weights keep PyTorch's default initialisation.
    The skips x1, x2, x3 are written by the trunk straight into the concat buffers' second slices and read from there by
    the next trunk stage; the x2 upsamplings write into the first slices (directly when no resample is needed)."""

    DECODER = (("conv1", 2048, 192), ("upconv1", 192, 128), ("conv2", 1152, 128), ("upconv2", 128, 96), ("conv3", 608, 96),
               ("upconv3", 96, 64), ("conv4", 320, 64), ("upconv4", 64, 48), ("conv5", 48, 48), ("upconv5", 48, 32),
               ("conv6", 32, 32))
    UP_CHANNELS = {3: 128, 2: 96, 1: 64}  # channels of the upsampled slice of the concat at skip x_i (upconv1, 2, 3)

    def __init__(self, num_classes, in_channels=3, backbone="resnet50", pretrained=None, freeze_bn=False, freeze_backbone=False,
                 **_):
        super().__init__()
        if backbone not in RESNET_BLOCKS:
            raise NotImplementedError(f"seg_b200.UNetResnet: backbone {backbone!r} not built (the decoder expects the 2048 "
                                      f"channels of resnet50/101/152)")
        _check_pretrained(self, pretrained)
        if in_channels != 3:
            raise NotImplementedError("in_channels != 3 swaps the deep stem for a 64-channel 7x7 conv that bn1 cannot take "
                                      "(unet.py:131-132); not built")
        self.num_classes = num_classes
        self.initial = _deep_stem()
        plan = [(1, 1, 1), (2, 1, 1), (1, 1, 2), (1, 2, 4)]  # resnet.py:190-210, as PSPNet
        self.layer1, self.layer2, self.layer3, self.layer4 = _res_layers(RESNET_BLOCKS[backbone], 128, plan)
        for name, cin, cout in self.DECODER:
            if name.startswith("up"):
                setattr(self, name, nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=False))
            else:
                setattr(self, name, nn.Conv2d(cin, cout, kernel_size=3, stride=1, padding=1))
        self.conv7 = nn.Conv2d(32, num_classes, kernel_size=1, bias=False)
        _init_like_reference_head(self)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(self.get_backbone_params())

    def _conv(self, tape, x, name):
        y, _ = tape.conv(x, self._spec(name, getattr(self, name)))
        return y

    def _up(self, tape, x, name, skip_hw, out):
        """upconvN (x2), resampled to the skip's size (bilinear, align_corners=True) unless it already has it, into `out`."""
        spec = self._spec(name, getattr(self, name))
        h, w = x.t.shape[1], x.t.shape[2]
        if (2 * h, 2 * w) == tuple(skip_hw):  # bilinear at equal size with align_corners=True is the identity
            return tape.conv_transpose(x, spec, out=out)
        return tape.bilinear(tape.conv_transpose(x, spec), skip_hw[0], skip_hw[1], True, out=out)

    def _forward_heads(self, tape, x):
        N, H, W = x.shape[0], x.shape[2], x.shape[3]
        dev = x.device
        a = self._stem(tape, x, "initial", self.initial)
        # concat buffers (upsampled, skip) at the sizes of x1, x2, x3: the last block of layers 1-3 writes its output into
        # the skip slice, and the next layer reads it from there
        cats, skips = {}, {}
        for li in (1, 2, 3, 4):
            layer = getattr(self, f"layer{li}")
            out = None
            if li < 4:
                s = layer[0].conv2.stride[0]
                h, w = (a.t.shape[1] - 1) // s + 1, (a.t.shape[2] - 1) // s + 1
                cout = layer[-1].conv3.out_channels
                cats[li] = tape.concat(N, h, w, [self.UP_CHANNELS[li], cout], dev)
                out = cats[li][1][1]
            for bi, blk in enumerate(layer):
                a = self._block(tape, a, f"layer{li}.{bi}.", blk, out=out if bi == len(layer) - 1 else None)
            if li < 4:
                skips[li] = a
        y = self._conv(tape, a, "conv1")
        for li, (up, conv) in zip((3, 2, 1), (("upconv1", "conv2"), ("upconv2", "conv3"), ("upconv3", "conv4"))):
            whole, sl = cats[li]
            skip = skips[li]
            u = self._up(tape, y, up, skip.t.shape[1:3], sl[0])
            tape.bind_slices(whole, [u, skip])
            tape.shared_slice(skip)  # the skip also feeds the next trunk layer: its two gradients add
            y = self._conv(tape, whole, conv)
        y = self._conv(tape, tape.conv_transpose(y, self._spec("upconv4", self.upconv4)), "conv5")
        y = tape.conv_transpose(y, self._spec("upconv5", self.upconv5))
        if (y.t.shape[1], y.t.shape[2]) != (H, W):  # unet.py:201-202
            y = tape.bilinear(y, H, W, True)
        y = self._conv(tape, y, "conv6")
        lo, _ = tape.conv(y, self._spec("conv7", self.conv7), out_dtype=torch.float32)
        return [FullResHead(lo)]

    def get_backbone_params(self):
        return chain(self.initial.parameters(), self.layer1.parameters(), self.layer2.parameters(), self.layer3.parameters(),
                     self.layer4.parameters())

    def get_decoder_params(self):
        return chain(*(getattr(self, n).parameters() for n, _, _ in self.DECODER), self.conv7.parameters())


# ----------------------------------------------------------------------------------------------- SegNet
def _vgg_stage(cin, widths):
    """(Conv2d 3x3 p1 with bias, BatchNorm2d, ReLU) per width: the nn.Sequential index layout of torchvision's vgg16_bn
    features, so that `stageN_encoder.3.weight` etc. line up with the reference."""
    mods = []
    for w in widths:
        mods += [nn.Conv2d(cin, w, kernel_size=3, stride=1, padding=1), nn.BatchNorm2d(w), nn.ReLU(inplace=True)]
        cin = w
    return nn.Sequential(*mods)


class SegNet(_EngineModel):
    """VGG16-BN encoder-decoder with max-pool indices — replaces models/segnet.py:13-132.  Encoder stages 64², 128², 256³,
    512³, 512³ (vgg16_bn's features without the pools); decoder stages 1-5 are the reversed encoder convs (9, 9, 9, 6 and 6
    modules) with the channel-changing ones rebuilt as 512->256, 256->128 and 128->64 plus a new BatchNorm, then
    `stage5_decoder.6` = Conv2d(64, num_classes, 3, p1).  Every conv has a bias.  Each encoder stage ends in
    MaxPool2d(2, 2, return_indices=True); each decoder stage starts with MaxUnpool2d(2, 2) to the size of the matching
    encoder map, so the logits are at input resolution for any input of at least 32 x 32 (smaller ones leave the fifth pool
    empty and raise ValueError).
    Init as the reference: the encoder keeps torchvision's VGG init (kaiming-normal fan_out convs, bias 0, BN 1 / 0; with
    in_channels != 3 `stage1_encoder.0` is a default-initialised Conv2d), the decoder gets kaiming-normal (fan_in) convs,
    bias 0, BN 1 / 0.  Parameter groups as the reference's: no backbone group, every parameter in the decoder group."""

    ENCODER = ((64, 64), (128, 128), (256, 256, 256), (512, 512, 512), (512, 512, 512))
    DECODER = ((512, (512, 512, 512)), (512, (512, 512, 256)), (256, (256, 256, 128)), (128, (128, 64)), (64, (64, 64)))
    MIN_SIZE = 32
    IM2COL_CONV = "stage1_encoder.0"

    def __init__(self, num_classes, in_channels=3, pretrained=None, freeze_bn=False, freeze_backbone=False, **_):
        super().__init__()
        _check_pretrained(self, pretrained)
        self.num_classes = num_classes
        cin = 3
        for i, widths in enumerate(self.ENCODER):
            setattr(self, f"stage{i + 1}_encoder", _vgg_stage(cin, widths))
            cin = widths[-1]
        for m in self.modules():  # torchvision VGG._initialize_weights (no weights: the reference's shimmed vgg16_bn)
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if in_channels != 3:
            self.stage1_encoder[0] = nn.Conv2d(in_channels, 64, kernel_size=3, stride=1, padding=1)
        self.pool = nn.MaxPool2d(kernel_size=2, stride=2, return_indices=True)  # holder: the engine runs Tape.maxpool2x2
        for i, (cin, widths) in enumerate(self.DECODER):
            setattr(self, f"stage{i + 1}_decoder", _vgg_stage(cin, widths))
        self.stage5_decoder.append(nn.Conv2d(64, num_classes, kernel_size=3, stride=1, padding=1))
        self.unpool = nn.MaxUnpool2d(kernel_size=2, stride=2)
        for i in range(1, 6):  # segnet.py:69-78
            for m in getattr(self, f"stage{i}_decoder").modules():
                if isinstance(m, nn.Conv2d):
                    nn.init.kaiming_normal_(m.weight)
                    m.bias.data.zero_()
                elif isinstance(m, nn.BatchNorm2d):
                    m.weight.data.fill_(1)
                    m.bias.data.zero_()
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(chain(*(getattr(self, f"stage{i}_encoder").parameters() for i in range(1, 6))))

    def _check_size(self, x):
        H, W = x.shape[-2], x.shape[-1]
        if H < self.MIN_SIZE or W < self.MIN_SIZE:
            raise ValueError(f"SegNet needs an input of at least {self.MIN_SIZE}x{self.MIN_SIZE} (five 2x2 max-pools); got {H}x{W}")

    def forward(self, x):
        self._check_size(x)
        return super().forward(x)

    def _stage(self, tape, a, name):
        seq = getattr(self, name)
        for j in range(0, len(seq) - len(seq) % 3, 3):  # (conv, BN, ReLU) triples; stage5_decoder.6 is the classifier
            a = self._cbr(tape, a, f"{name}.{j}", seq[j], seq[j + 1])
        return a

    def _forward_heads(self, tape, x):
        self._check_size(x)
        a, records = x, []
        for i in range(1, 6):
            a, rec = tape.maxpool2x2(self._stage(tape, a, f"stage{i}_encoder"))
            records.append(rec)
        for i in range(1, 6):
            a = self._stage(tape, tape.maxunpool2x2(a, records[5 - i]), f"stage{i}_decoder")
        lo, _ = tape.conv(a, self._spec("stage5_decoder.6", self.stage5_decoder[6]), out_dtype=torch.float32)
        return [FullResHead(lo)]

    def get_backbone_params(self):
        return []

    def get_decoder_params(self):
        return self.parameters()


# ----------------------------------------------------------------------------------------------- FCN8
def upsampling_weight(in_channels, out_channels, kernel_size):
    """The bilinear ConvTranspose2d init of utils/helpers.py:get_upsampling_weight: the separable tent filter on the channel
    diagonal, zeros elsewhere."""
    factor = (kernel_size + 1) // 2
    center = factor - 1 if kernel_size % 2 == 1 else factor - 0.5
    og = np.ogrid[:kernel_size, :kernel_size]
    filt = (1 - abs(og[0] - center) / factor) * (1 - abs(og[1] - center) / factor)
    weight = np.zeros((in_channels, out_channels, kernel_size, kernel_size), dtype=np.float64)
    weight[list(range(in_channels)), list(range(out_channels)), :, :] = filt
    return torch.from_numpy(weight).float()


class FCN8(_EngineModel):
    """FCN-8s on a VGG16 trunk — replaces models/fcn.py:9-103 (which cannot be constructed: it reads an undefined
    `freeze_backbone`).  pool3 / pool4 / pool5 = torchvision vgg16().features[:17] / [17:24] / [24:] with the first conv padded
    by 100 and every MaxPool2d in ceil mode; output = conv6 (7x7, 512 -> 4096) ReLU Dropout conv7 (1x1) ReLU Dropout
    Conv2d(4096, C, 1); adj_pool3 / adj_pool4 = 1x1 convs to C; up_output / up_pool4_out = ConvTranspose2d(C, C, 4, 2) and
    up_final = ConvTranspose2d(C, C, 16, 8), bias-free, bilinear-initialised and frozen.
    Forward: each conv runs on the wgmma kernels with its bias in the epilogue, the ReLU standalone or fused with the stage's
    ceil-mode pool (`Tape.relu_maxpool_ceil`), conv6 / conv7's ReLU + Dropout in one pass.  The adj convs write W·pool
    without their bias; each upsampler is one `Tape.score_upsample` launch over only its cropped window, adding
    alpha * skip + bias (alpha = 0.01, 1e-4) in the same pass, so s2, s4 (bf16) and the cropped fp32 logits come out of one
    launch each.
    Init as the reference: torchvision's VGG init for the features (kaiming-normal fan_out, bias 0), conv6 / conv7 from
    N(0, 0.01) Linear weights with bias 0, default init for the score and adj convs.  Parameter groups as the reference's.
    freeze_backbone freezes pool3 / pool4 / pool5.  An input with other than 3 channels raises ValueError."""

    VGG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")

    def __init__(self, num_classes, pretrained=None, freeze_bn=False, freeze_backbone=False, **_):
        super().__init__()
        _check_pretrained(self, pretrained)
        self.num_classes = num_classes
        features, cin = [], 3
        for v in self.VGG:
            if v == "M":
                features.append(nn.MaxPool2d(kernel_size=2, stride=2, ceil_mode=True))
            else:
                features += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
                cin = v
        features[0].padding = (100, 100)
        for m in features:  # torchvision VGG._initialize_weights
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                nn.init.constant_(m.bias, 0)
        self.pool3 = nn.Sequential(*features[:17])
        self.pool4 = nn.Sequential(*features[17:24])
        self.pool5 = nn.Sequential(*features[24:])
        self.adj_pool3 = nn.Conv2d(256, num_classes, kernel_size=1)
        self.adj_pool4 = nn.Conv2d(512, num_classes, kernel_size=1)
        conv6 = nn.Conv2d(512, 4096, kernel_size=7)
        conv7 = nn.Conv2d(4096, 4096, kernel_size=1)
        for c in (conv6, conv7):  # vgg.classifier[0] / [3]: nn.Linear with torchvision's N(0, 0.01), bias 0, reshaped
            nn.init.normal_(c.weight, 0, 0.01)
            nn.init.constant_(c.bias, 0)
        self.output = nn.Sequential(conv6, nn.ReLU(inplace=True), nn.Dropout(), conv7, nn.ReLU(inplace=True), nn.Dropout(),
                                    nn.Conv2d(4096, num_classes, kernel_size=1))
        self.up_output = nn.ConvTranspose2d(num_classes, num_classes, kernel_size=4, stride=2, bias=False)
        self.up_pool4_out = nn.ConvTranspose2d(num_classes, num_classes, kernel_size=4, stride=2, bias=False)
        self.up_final = nn.ConvTranspose2d(num_classes, num_classes, kernel_size=16, stride=8, bias=False)
        for up, k in ((self.up_output, 4), (self.up_pool4_out, 4), (self.up_final, 16)):
            up.weight.data.copy_(upsampling_weight(num_classes, num_classes, k))
            up.weight.requires_grad = False
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            _freeze(chain(self.pool3.parameters(), self.pool4.parameters(), self.pool5.parameters()))

    def all_conv_specs(self):
        # the frozen upsamplers run on the score kernels, not the conv path: no packed weight or weight gradient
        return [self._spec(n, m) for n, m in self.named_modules() if isinstance(m, nn.Conv2d)]

    def _check(self, x):
        """Before any launch: a 3-channel NCHW input, and frozen upsamplers (the engine computes no gradient for them)."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"FCN8 takes a 3-channel NCHW input (VGG16's first conv); got shape {tuple(x.shape)}")
        for name in ("up_output", "up_pool4_out", "up_final"):
            if getattr(self, name).weight.requires_grad:
                raise NotImplementedError(f"FCN8.{name}: the engine computes no gradient for the upsampling weight; keep it "
                                          "frozen (requires_grad=False), as models/fcn.py does")

    def forward(self, x):
        self._check(x)
        return super().forward(x)

    def _forward_heads(self, tape, x):
        self._check(x)
        N, _, H, W = x.shape
        a, taps = x, []
        for name in ("pool3", "pool4", "pool5"):
            seq = getattr(self, name)
            for j, m in enumerate(seq):
                if isinstance(m, nn.Conv2d):
                    y, _ = tape.conv(a, self._spec(f"{name}.{j}", m))
                    pool_next = j + 2 < len(seq) and isinstance(seq[j + 2], nn.MaxPool2d)
                    a = tape.relu_maxpool_ceil(y) if pool_next else tape.relu(y)
            taps.append(a)
        pool3, pool4, pool5 = taps
        out, C, dev = self.output, self.num_classes, x.device
        a = tape.relu_dropout(tape.conv(pool5, self._spec("output.0", out[0]))[0], out[2].p)
        a = tape.relu_dropout(tape.conv(a, self._spec("output.3", out[3]))[0], out[5].p)
        _, h, w, _ = a.t.shape
        score, _ = tape.conv(a, self._spec("output.6", out[6]), out=tape.pitched(N, h, w, C, dev))
        # s2 = adj_pool4(0.01 * pool4)[5:5+h2, 5:5+w2] + up_output(score)  (fcn.py:85-88)
        skip4, _ = tape.conv(pool4, self._spec("adj_pool4", self.adj_pool4), out=tape.pitched(N, *pool4.shape[1:3], C, dev),
                             use_bias=False)
        h2, w2 = 2 * h + 2, 2 * w + 2
        s2 = tape.score_upsample(score, self.up_output, (0, 0, h2, w2), skip=skip4, skip_off=(5, 5), alpha=0.01,
                                 bias=self.adj_pool4.bias)
        # s4 = adj_pool3(0.0001 * pool3)[9:9+h4, 9:9+w4] + up_pool4_out(s2)  (fcn.py:91-92)
        skip3, _ = tape.conv(pool3, self._spec("adj_pool3", self.adj_pool3), out=tape.pitched(N, *pool3.shape[1:3], C, dev),
                             use_bias=False)
        h4, w4 = 2 * h2 + 2, 2 * w2 + 2
        s4 = tape.score_upsample(s2, self.up_pool4_out, (0, 0, h4, w4), skip=skip3, skip_off=(9, 9), alpha=1e-4,
                                 bias=self.adj_pool3.bias)
        # logits = up_final(s4)[31:31+H, 31:31+W]  (fcn.py:95-96)
        lo = tape.score_upsample(s4, self.up_final, (31, 31, H, W), out_dtype=torch.float32)
        return [FullResHead(lo)]

    def get_backbone_params(self):
        return chain(self.pool3.parameters(), self.pool4.parameters(), self.pool5.parameters(), self.output.parameters())

    def get_decoder_params(self):
        return chain(self.up_output.parameters(), self.adj_pool4.parameters(), self.up_pool4_out.parameters(),
                     self.adj_pool3.parameters(), self.up_final.parameters())


# ----------------------------------------------------------------------------------------------- PSPDenseNet
DENSENET_BLOCKS = {"densenet121": (6, 12, 24, 16), "densenet169": (6, 12, 32, 32), "densenet201": (6, 12, 48, 32)}
GROWTH, BN_SIZE = 32, 4  # torchvision densenet121/169/201: growth_rate 32, bn_size 4, num_init_features 64


def _dense_block(cin, n, dil):
    """torchvision _DenseBlock holder: denselayerK = norm1, relu1, conv1 (1x1 -> 4 * growth), norm2, relu2, conv2 (3x3 ->
    growth, dilation / padding `dil`), reading the concat of the block input and every earlier layer's output."""
    blk = _Holder()
    for k in range(n):
        lay = _Holder()
        lay.norm1, lay.relu1 = nn.BatchNorm2d(cin + k * GROWTH), nn.ReLU(inplace=True)
        lay.conv1 = nn.Conv2d(cin + k * GROWTH, BN_SIZE * GROWTH, 1, bias=False)
        lay.norm2, lay.relu2 = nn.BatchNorm2d(BN_SIZE * GROWTH), nn.ReLU(inplace=True)
        lay.conv2 = nn.Conv2d(BN_SIZE * GROWTH, GROWTH, 3, padding=dil, dilation=dil, bias=False)
        setattr(blk, f"denselayer{k + 1}", lay)
    return blk


class PSPDenseNet(_EngineModel):
    """PSPNet over a dilated DenseNet-121/169/201 — replaces models/pspnet.py:117-205 (trained from scratch: the custom
    block0).  block0 = Conv2d(in, 64, 3, s2) BN ReLU, then [Conv2d(64, 64, 3) BN ReLU] * 2 — ONE conv and ONE BN applied
    twice (block0.3 is block0.6, block0.4 is block0.7; every conv unpadded), MaxPool2d(3, 2, 1); the dense blocks; transition1
    = norm relu 1x1 conv AvgPool2d(2, 2); transition2 / 3 without the pool; block3 / block4's conv2 dilated 2 / 4; no norm5:
    block4's concat feeds the PSP module (bins 1, 2, 3, 6), whose bottleneck, dropout and classifier are PSPNet's; the aux
    branch reads transition3's output.  Logits: bilinear, align_corners=False.
    Each dense block is ONE buffer of its final width (`Tape.dense_buffer`): the block input and every conv2 write their
    channel slice in place, and each norm1 is a pre-activation BN over the prefix, whose batch statistics come from the
    block's table of per-slice records (`Tape.bn_act(table=)`) and whose backward adds into the prefix of the block's
    gradient.  block4's buffer is the PSP concat, so the trunk output is never copied.
    Init as the reference: torchvision's DenseNet init for the trunk (kaiming-normal convs, BN 1 / 0), initialize_weights for
    block0 and the heads.  Parameter groups as the reference's (block4 is in neither).  freeze_backbone is ignored, as
    there.  densenet161 raises NotImplementedError: its block1 expects 96 channels and the reference cannot train it from
    scratch."""

    IM2COL_CONV = "block0.0"

    def __init__(self, num_classes, in_channels=3, backbone="densenet201", pretrained=None, use_aux=True, freeze_bn=False, **_):
        super().__init__()
        if backbone == "densenet161":
            raise NotImplementedError("PSPDenseNet(densenet161) cannot train from scratch in the reference either: its block1 "
                                      "expects 96 input channels but block0 gives 64 (RuntimeError: running_mean should "
                                      "contain 64 elements not 96)")
        if backbone not in DENSENET_BLOCKS:
            raise NotImplementedError(f"seg_b200.PSPDenseNet: backbone {backbone!r} not built")
        _check_pretrained(self, pretrained)
        self.num_classes, self.use_aux = num_classes, use_aux
        self.layers = DENSENET_BLOCKS[backbone]
        c3 = nn.Conv2d(64, 64, 3, bias=False)
        n3 = nn.BatchNorm2d(64)
        r3 = nn.ReLU(inplace=True)
        self.block0 = nn.Sequential(nn.Conv2d(in_channels, 64, 3, stride=2, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
                                    c3, n3, r3, c3, n3, r3, nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        widths, c = [], 64
        for bi, n in enumerate(self.layers):
            widths.append((c, c + n * GROWTH))
            c = (c + n * GROWTH) // 2
        self.widths = widths  # (input, output) channels of each dense block
        for bi, ((cin, _), n, dil) in enumerate(zip(widths, self.layers, (1, 1, 2, 4))):
            setattr(self, f"block{bi + 1}", _dense_block(cin, n, dil))
        t1 = _Holder()
        t1.norm, t1.relu = nn.BatchNorm2d(widths[0][1]), nn.ReLU(inplace=True)
        t1.conv = nn.Conv2d(widths[0][1], widths[1][0], 1, bias=False)
        t1.pool = nn.AvgPool2d(kernel_size=2, stride=2)
        self.transition1 = t1
        for k in (2, 3):
            cin, cout = widths[k - 1][1], widths[k][0]
            setattr(self, f"transition{k}", nn.Sequential(nn.BatchNorm2d(cin), nn.ReLU(inplace=True), nn.Conv2d(cin, cout, 1, bias=False)))
        self.master_branch, self.auxiliary_branch = _psp_branches(widths[3][1], widths[3][0], num_classes)
        for mod in (self.block1, self.block2, self.block3, self.block4, self.transition1, self.transition2, self.transition3):
            for m in mod.modules():  # torchvision DenseNet.__init__
                if isinstance(m, nn.Conv2d):
                    nn.init.kaiming_normal_(m.weight)
                elif isinstance(m, nn.BatchNorm2d):
                    nn.init.constant_(m.weight, 1)
                    nn.init.constant_(m.bias, 0)
        _init_like_reference_head(self.block0)
        _init_like_reference_head(self.master_branch, self.auxiliary_branch)
        if freeze_bn:
            self.freeze_bn()

    def _dense(self, tape, buf, table, bi, c0, dil):
        """Block bi's layers over its buffer (slice [0, c0) already written, its record in table[:2 c0])."""
        blk = getattr(self, f"block{bi}")
        for k in range(self.layers[bi - 1]):
            lay = getattr(blk, f"denselayer{k + 1}")
            cin, name = c0 + k * GROWTH, f"block{bi}.denselayer{k + 1}"
            h = tape.bn_act(tape.prefix(buf, 0, cin), lay.norm1, table=(table, c0, GROWTH))
            h = self._cbr(tape, h, name + ".conv1", lay.conv1, lay.norm2)
            rec = table[2 * cin:2 * cin + 2 * GROWTH] if table is not None else None
            y, _ = tape.conv(h, self._spec(name + ".conv2", lay.conv2), out=buf.t[..., cin:cin + GROWTH], want_stats=True,
                             stats_out=rec)
            tape.prefix(buf, cin, cin + GROWTH, act=y)

    def _block_buffer(self, tape, N, H, W, bi, pitch=None):
        c0, c1 = self.widths[bi - 1]
        buf = tape.dense_buffer(N, H, W, pitch or c1, self.block0[0].weight.device)
        table = tape.zalloc64(2 * c1, buf.t.device) if tape.training else None
        return buf, table

    def _forward_heads(self, tape, x):
        N, _, H, W = x.shape
        b0 = self.block0
        a = self._cbr(tape, x, "block0.0", b0[0], b0[1])
        a = self._cbr(tape, a, "block0.3", b0[3], b0[4])
        a = self._cbr(tape, a, "block0.3", b0[6], b0[7])  # block0.6 / block0.7 are block0.3 / block0.4: one ConvSpec
        a = tape.maxpool(a)
        Hb, Wb = a.t.shape[1], a.t.shape[2]
        # block1: the max-pooled stem is copied into slice 0
        buf, table = self._block_buffer(tape, N, Hb, Wb, 1)
        s0 = tape.prefix(buf, 0, 64, act=tape.copy_into(a, buf.t[..., :64]))
        if table is not None:
            tape.record_stats(s0, table[:128])
        self._dense(tape, buf, table, 1, 64, 1)
        # transition1: BN ReLU 1x1 conv, then the 2x2 average pool straight into block2's slice 0
        t1 = self.transition1
        h = tape.bn_act(buf, t1.norm, table=(table, 64, GROWTH))
        y, _ = tape.conv(h, self._spec("transition1.conv", t1.conv))
        c0 = self.widths[1][0]
        buf, table = self._block_buffer(tape, N, y.t.shape[1] // 2, y.t.shape[2] // 2, 2)
        s0 = tape.prefix(buf, 0, c0, act=tape.avgpool2x2(y, out=buf.t[..., :c0]))
        if table is not None:
            tape.record_stats(s0, table[:2 * c0])
        self._dense(tape, buf, table, 2, c0, 1)
        # transition2 / transition3: BN ReLU 1x1 conv straight into slice 0 of the next block (block4's is the PSP concat)
        m_out = self.widths[3][1]
        for bi, dil in ((3, 2), (4, 4)):
            tr = getattr(self, f"transition{bi - 1}")
            prev_c0 = self.widths[bi - 2][0]
            h = tape.bn_act(buf, tr[0], table=(table, prev_c0, GROWTH))
            c0 = self.widths[bi - 1][0]
            nbuf, ntable = self._block_buffer(tape, N, buf.t.shape[1], buf.t.shape[2], bi, pitch=2 * m_out if bi == 4 else None)
            y, _ = tape.conv(h, self._spec(f"transition{bi - 1}.2", tr[2]), out=nbuf.t[..., :c0], want_stats=True,
                             stats_out=ntable[:2 * c0] if ntable is not None else None)
            x_aux = tape.prefix(nbuf, 0, c0, act=y)
            buf, table = nbuf, ntable
            self._dense(tape, buf, table, bi, c0, dil)
        heads = []
        if self.training and self.use_aux:
            # recorded before the PSP head: in the backward the bottleneck's dgrad writes block4's gradient first (beta = 0),
            # then the aux conv adds into transition3's slice
            ab = self.auxiliary_branch
            ya = self._cbr(tape, x_aux, "auxiliary_branch.0", ab[0], ab[1], drop_p=ab[3].p, drop_channelwise=True)
            la, _ = tape.conv(ya, self._spec("auxiliary_branch.4", ab[4]), out_dtype=torch.float32)
            heads.append(BilinearHead(la, False, H, W))
        mb = self.master_branch
        y = self._ppm(tape, tape.prefix(buf, 0, m_out), mb[0], "master_branch.0", cat=buf)
        lo, _ = tape.conv(y, self._spec("master_branch.1", mb[1]), out_dtype=torch.float32)
        return [BilinearHead(lo, False, H, W)] + heads

    def get_backbone_params(self):
        return chain(self.block0.parameters(), self.block1.parameters(), self.block2.parameters(), self.block3.parameters(),
                     self.transition1.parameters(), self.transition2.parameters(), self.transition3.parameters())

    def get_decoder_params(self):
        return chain(self.master_branch.parameters(), self.auxiliary_branch.parameters())
