"""H100-native drop-in models for the reference's plugin surface (models/__init__.py registry):

    DeepLab(num_classes, in_channels=3, backbone='xception',  pretrained=None, output_stride=16, freeze_bn=False, **_)
    PSPNet (num_classes, in_channels=3, backbone='resnet152', pretrained=None, use_aux=True,   freeze_bn=False, **_)
    UperNet(num_classes, in_channels=3, backbone='resnet101', pretrained=None, use_aux=True, fpn_out=256, freeze_bn=False, **_)

(default backbones are the reference's; `pretrained`: the reference defaults to True and downloads ImageNet weights — there is
no network here, so an explicit True raises and the default (None) initialises randomly with a logged warning)

Same constructor contract, same `state_dict()` keys and OIHW fp32 parameter layout, same `get_backbone_params /
get_decoder_params / freeze_bn` methods and the same forward contract (fp32 NCHW logits at input resolution; PSPNet
returns `(out, aux)` in training) as models/deeplabv3_plus.py:336-377 and models/pspnet.py:41-105 — so train.py,
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
from .engine import Act, ConvSpec, DwSpec, Tape
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
    """plan: per layer (first-block stride, first-block dilation, other-block dilation)."""
    layers = []
    for li, (n, planes) in enumerate(zip(blocks, (64, 128, 256, 512))):
        stride, d0, d = plan[li]
        seq = []
        for b in range(n):
            seq.append(_bottleneck(inplanes, planes, stride if b == 0 else 1, d0 if b == 0 else d, b == 0))
            inplanes = planes * 4
        layers.append(nn.Sequential(*seq))
    return layers


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
        for (lo_act, Hl, Wl, ac), dout in zip(ctx.heads, douts):
            if dout is None:
                continue
            C = dout.shape[1]
            ldx = (C + 7) // 8 * 8
            g = ops.bilinear_logits_bwd(dout.contiguous().float(), Hl, Wl, ac, ldx)
            lo_act.grad = g[..., :C]
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
                for (lo_act, Hl, Wl, ac), d in zip(heads, e.douts):
                    C = d.shape[1]
                    g = ops.bilinear_logits_bwd(d, Hl, Wl, ac, (C + 7) // 8 * 8)
                    lo_act.grad = g[..., :C]
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
            s = ConvSpec(name, module)
            self._specs[name] = s
        return s

    def all_conv_specs(self):
        """ConvSpec of every dense nn.Conv2d holder (names = module paths, as used by the forward code)."""
        return [self._spec(n, m) for n, m in self.named_modules() if isinstance(m, nn.Conv2d) and m.groups == 1]

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

    def _block(self, tape, x, prefix, blk):
        a = self._cbr(tape, x, prefix + "conv1", blk.conv1, blk.bn1)
        a = self._cbr(tape, a, prefix + "conv2", blk.conv2, blk.bn2)
        r = x
        if blk.downsample is not None:
            r = self._cbr(tape, x, prefix + "downsample.0", blk.downsample[0], blk.downsample[1], relu=False)
        return self._cbr(tape, a, prefix + "conv3", blk.conv3, blk.bn3, relu=True, res=r)

    def _finish(self, tape):
        if tape.bn_modules:
            torch._foreach_add_([m.num_batches_tracked for m in tape.bn_modules], 1)

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
        H, W = x.shape[2], x.shape[3]
        tape = self._new_tape(training, record)
        if tables is not None:  # graph capture: persistent packed weights / packed weight-gradient accumulators
            tape.packed_override, tape.dw_buffers = tables.packed_bufs, tables.dw_bufs
        if grads is not None:
            tape.grads = dict(grads)  # pre-bound views: every parameter gradient lands in one flat buffer
        heads = self._forward_heads(tape, x)
        outs = tuple(ops.bilinear_logits_fwd(lo.t, H, W, ac) for lo, ac in heads)
        self._finish(tape)
        return outs, tape, [(lo, lo.t.shape[1], lo.t.shape[2], ac) for lo, ac in heads]

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
            if freeze_bn:
                self.freeze_bn()
            if freeze_backbone:
                for p in self.backbone.parameters():
                    p.requires_grad = False
            return
        # deeplabv3_plus.py:35-53: os16 -> layer3 stride 2, layer4 every conv2 d=2 ; os8 -> layer3 d=2, layer4 d=4
        if output_stride == 16:
            plan = [(1, 1, 1), (2, 1, 1), (2, 1, 1), (1, 2, 2)]
        else:
            plan = [(1, 1, 1), (2, 1, 1), (1, 2, 2), (1, 4, 4)]
        bb = _Holder()
        c0, b0 = nn.Conv2d(in_channels, 64, 7, stride=2, padding=3, bias=False), nn.BatchNorm2d(64)
        bb.layer0 = nn.Sequential(c0, b0, nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        bb.layer1, bb.layer2, bb.layer3, bb.layer4 = _res_layers(RESNET_BLOCKS[backbone], 64, plan)
        self.backbone = bb
        self._build_heads(num_classes, output_stride, low_level_channels=256)
        _init_like_torchvision_trunk(bb.layer1, bb.layer2, bb.layer3, bb.layer4)
        _init_like_reference_head(bb.layer0, self.ASSP, self.decoder)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            for p in self.backbone.parameters():
                p.requires_grad = False

    def _build_heads(self, num_classes, output_stride, low_level_channels):
        dil = (1, 6, 12, 18) if output_stride == 16 else (1, 12, 24, 36)
        a = _Holder()
        for i, k in zip((1, 2, 3, 4), (1, 3, 3, 3)):
            c, n = _cbn(2048, 256, k, 1, dil[i - 1])
            setattr(a, f"aspp{i}", nn.Sequential(c, n, nn.ReLU(inplace=True)))
        c, n = _cbn(2048, 256, 1)
        a.avg_pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), c, n, nn.ReLU(inplace=True))
        a.conv1, a.bn1 = _cbn(256 * 5, 256, 1)
        a.relu, a.dropout = nn.ReLU(inplace=True), nn.Dropout(0.5)
        self.ASSP = a
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

    def _trunk_resnet(self, tape, x):
        bb = self.backbone
        a = self._cbr(tape, x, "backbone.layer0.0", bb.layer0[0], bb.layer0[1])
        a = tape.maxpool(a)
        low = None
        for li in (1, 2, 3, 4):
            layer = getattr(bb, f"layer{li}")
            for bi, blk in enumerate(layer):
                a = self._block(tape, a, f"backbone.layer{li}.{bi}.", blk)
            if li == 1:
                low = a
        return a, low

    def _aspp(self, tape, a):
        """ASSP.forward (deeplabv3_plus.py:286-297): five branches written straight into one 1280-channel buffer."""
        N, Hf, Wf = a.t.shape[0], a.t.shape[1], a.t.shape[2]
        A = self.ASSP
        cat, sl = tape.concat(N, Hf, Wf, [256] * 5, a.t.device)
        br = []
        for i in (1, 2, 3, 4):
            seq = getattr(A, f"aspp{i}")
            br.append(self._cbr(tape, a, f"ASSP.aspp{i}.0", seq[0], seq[1], out=sl[i - 1]))
        g = tape.avgpool(a, 1)
        g = self._cbr(tape, g, "ASSP.avg_pool.1", A.avg_pool[1], A.avg_pool[2])
        br.append(tape.bilinear(g, Hf, Wf, True, out=sl[4]))
        tape.bind_slices(cat, br)
        return self._cbr(tape, cat, "ASSP.conv1", A.conv1, A.bn1, drop_p=A.dropout.p)

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
        a, low = self._trunk_xception(tape, x) if self.backbone_name == "xception" else self._trunk_resnet(tape, x)
        return self._decoder(tape, self._aspp(tape, a), low)

    def _forward_heads(self, tape, x):
        """[(stride-4 fp32 logits Act, align_corners of the final upsample)]  (deeplabv3_plus.py:361: True)"""
        return [(self._features(tape, x), True)]

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
        s1, n1 = _cbn(3, 64, 3, 2, 1)
        s2, n2 = _cbn(64, 64, 3, 1, 1)
        s3 = nn.Conv2d(64, 128, 3, stride=1, padding=1, bias=False)
        stem = nn.Sequential(s1, n1, nn.ReLU(inplace=True), s2, n2, nn.ReLU(inplace=True), s3)
        self.initial = nn.Sequential(stem, nn.BatchNorm2d(128), nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        # resnet.py:154-163,190-210: layer3 = [d1, d2, ...], layer4 = [d2, d4, ...], all stride 1 (output stride 8)
        plan = [(1, 1, 1), (2, 1, 1), (1, 1, 2), (1, 2, 4)]
        self.layer1, self.layer2, self.layer3, self.layer4 = _res_layers(RESNET_BLOCKS[backbone], 128, plan)
        m_out = 2048
        psp = _Holder()
        stages = []
        for b in (1, 2, 3, 6):
            c, n = _cbn(m_out, m_out // 4, 1)
            stages.append(nn.Sequential(nn.AdaptiveAvgPool2d(output_size=b), c, n, nn.ReLU(inplace=True)))
        psp.stages = nn.ModuleList(stages)
        c, n = _cbn(m_out * 2, m_out // 4, 3)
        psp.bottleneck = nn.Sequential(c, n, nn.ReLU(inplace=True), nn.Dropout2d(0.1))
        self.master_branch = nn.Sequential(psp, nn.Conv2d(m_out // 4, num_classes, kernel_size=1))
        c, n = _cbn(m_out // 2, m_out // 4, 3)
        self.auxiliary_branch = nn.Sequential(c, n, nn.ReLU(inplace=True), nn.Dropout2d(0.1),
                                              nn.Conv2d(m_out // 4, num_classes, kernel_size=1))
        self.bins = (1, 2, 3, 6)
        _init_like_resnet_s(self.initial, self.layer1, self.layer2, self.layer3, self.layer4)
        _init_like_reference_head(self.master_branch, self.auxiliary_branch)
        if freeze_bn:
            self.freeze_bn()
        if freeze_backbone:
            for m in (self.initial, self.layer1, self.layer2, self.layer3, self.layer4):
                for p in m.parameters():
                    p.requires_grad = False

    def _forward_heads(self, tape, x):
        N = x.shape[0]
        stem = self.initial[0]
        a = self._cbr(tape, x, "initial.0.0", stem[0], stem[1])
        a = self._cbr(tape, a, "initial.0.3", stem[3], stem[4])
        a = self._cbr(tape, a, "initial.0.6", stem[6], self.initial[1])
        a = tape.maxpool(a)
        x_aux = None
        for li in (1, 2, 3, 4):
            for bi, blk in enumerate(getattr(self, f"layer{li}")):
                a = self._block(tape, a, f"layer{li}.{bi}.", blk)
            if li == 3:
                x_aux = a
        lo = self._psp_head(tape, a)
        heads = [(lo, False)]  # pspnet.py:86,91: F.interpolate default align_corners=False; the crop is a no-op
        if self.training and self.use_aux:
            ab = self.auxiliary_branch
            ya = self._cbr(tape, x_aux, "auxiliary_branch.0", ab[0], ab[1], drop_p=ab[3].p, drop_channelwise=True)
            la, _ = tape.conv(ya, self._spec("auxiliary_branch.4", ab[4]), out_dtype=torch.float32)
            heads.append((la, False))
        return heads

    def _psp_head(self, tape, a):
        """_PSPModule.forward + the classifier (pspnet.py:31-38, :66-70): returns the fp32 stride-8 logits Act."""
        N, Hf, Wf = a.t.shape[0], a.t.shape[1], a.t.shape[2]
        psp = self.master_branch[0]
        # pspnet.py:31-38: cat([features, stage1..4]) -> 3x3 bottleneck.  The trunk output is copied into slice 0
        # (it is also the residual-stream tensor, so it cannot simply be produced in place there).
        cat, sl = tape.concat(N, Hf, Wf, [2048, 512, 512, 512, 512], a.t.device)
        feats = tape.copy_into(a, sl[0])
        br = [feats]
        for i, b in enumerate(self.bins):
            st = psp.stages[i]
            p = tape.avgpool(a, b)
            p = self._cbr(tape, p, f"master_branch.0.stages.{i}.1", st[1], st[2])
            br.append(tape.bilinear(p, Hf, Wf, True, out=sl[i + 1]))
        tape.bind_slices(cat, br)
        y = self._cbr(tape, cat, "master_branch.0.bottleneck.0", psp.bottleneck[0], psp.bottleneck[1], drop_p=psp.bottleneck[3].p,
                      drop_channelwise=True)
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
        c0, b0 = nn.Conv2d(in_channels, 64, 7, stride=2, padding=3, bias=False), nn.BatchNorm2d(64)
        bb.initial = nn.Sequential(c0, b0, nn.ReLU(inplace=True), nn.MaxPool2d(kernel_size=3, stride=2, padding=1))
        bb.layer1, bb.layer2, bb.layer3, bb.layer4 = _res_layers(RESNET_BLOCKS[backbone], 64, [(1, 1, 1), (2, 1, 1), (2, 1, 1), (1, 2, 2)])
        self.backbone = bb
        feats = [256, 512, 1024, 2048]
        ppn = _Holder()
        self.bins = (1, 2, 4, 6)
        stages = []
        for b in self.bins:
            c, n = _cbn(feats[-1], feats[-1] // 4, 1)
            stages.append(nn.Sequential(nn.AdaptiveAvgPool2d(output_size=b), c, n, nn.ReLU(inplace=True)))
        ppn.stages = nn.ModuleList(stages)
        c, n = _cbn(feats[-1] * 2, feats[-1], 3)
        ppn.bottleneck = nn.Sequential(c, n, nn.ReLU(inplace=True), nn.Dropout2d(0.1))
        self.PPN = ppn
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
            for p in self.backbone.parameters():
                p.requires_grad = False

    def _forward_heads(self, tape, x):
        N = x.shape[0]
        bb = self.backbone
        a = self._cbr(tape, x, "backbone.initial.0", bb.initial[0], bb.initial[1])
        a = tape.maxpool(a)
        feats = []
        for li in (1, 2, 3, 4):
            for bi, blk in enumerate(getattr(bb, f"layer{li}")):
                a = self._block(tape, a, f"backbone.layer{li}.{bi}.", blk)
            feats.append(a)
        # ---- PPN on the last feature map (upernet.py:31-38) ----
        f4 = feats[-1]
        Hf, Wf = f4.t.shape[1], f4.t.shape[2]
        cat, sl = tape.concat(N, Hf, Wf, [2048, 512, 512, 512, 512], f4.t.device)
        br = [tape.copy_into(f4, sl[0])]
        for i, b in enumerate(self.bins):
            st = self.PPN.stages[i]
            p = tape.avgpool(f4, b)
            p = self._cbr(tape, p, f"PPN.stages.{i}.1", st[1], st[2])
            br.append(tape.bilinear(p, Hf, Wf, True, out=sl[i + 1]))
        tape.bind_slices(cat, br)
        pb = self.PPN.bottleneck
        feats[-1] = self._cbr(tape, cat, "PPN.bottleneck.0", pb[0], pb[1], drop_p=pb[3].p, drop_channelwise=True)
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
        return [(lo, False)]  # upernet.py:143: F.interpolate default align_corners=False

    def get_backbone_params(self):
        return self.backbone.parameters()

    def get_decoder_params(self):
        return chain(self.PPN.parameters(), self.FPN.parameters(), self.head.parameters())
